// fm_context.cu -- the C ABI declared in include/fmb200.h: context lifetime,
// host<->HBM layout conversion (bit-exact index/ordering work), epoch /
// evaluate / predict entry points.  CUDA only: no CPU fallback exists.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>

#include "fmb200_internal.h"

using namespace fmb;

namespace {

thread_local char g_err[512] = "";

int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

#define CK(expr)                                                                      \
  do {                                                                                \
    cudaError_t e__ = (expr);                                                         \
    if (e__ != cudaSuccess)                                                           \
      return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, \
                  __LINE__);                                                          \
  } while (0)

#define NEED_CTX(c) \
  if ((c) == nullptr) return fail("null context")

// No C++ exception may cross the C ABI: entry points that allocate host staging run
// their body through this.
template <class F>
int guarded(F&& body) {
  try {
    return body();
  } catch (const std::bad_alloc&) {
    return fail("out of host memory");
  } catch (...) {
    return fail("unexpected C++ exception");
  }
}

int bind(fmb200_ctx* c) {
  CK(cudaSetDevice(c->device));
  return 0;
}

// Make `slot` ready to receive a data set of (n_rows, nnz): drain an earlier asynchronous
// upload, (re)allocate, reset the bookkeeping.  Enqueues only the memsets of fresh buffers.
int upload_begin(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, cudaStream_t st) {
  DataSlot& s = c->slots[slot];
  if (s.pending) {  // an earlier asynchronous upload into this slot: drain it first
    CK(cudaEventSynchronize(s.ready.get()));
    s.pending = false;
  }
  // re-uploads into a slot reuse its buffers when they are large enough
  if (!(s.row_ptr && s.cap_rows >= n_rows && s.cap_nnz >= nnz)) {
    s = DataSlot();  // releases the slot's buffers, its ORDERED index and the index scratch
    CK(alloc(s.row_ptr, n_rows + 1 + kRowSlack));
    CK(alloc(s.target, n_rows + kRowSlack));
    CK(alloc(s.col, nnz + kEntrySlack));
    CK(alloc(s.val, nnz + kEntrySlack));
    CK(alloc(s.feat_cnt, c->n));
    CK(alloc(s.d_flag, 16));
    CK(host_alloc(s.h_flag, 16));
    CK(event_create(s.ready, cudaEventDisableTiming));
    // the slack is only ever read by whole-tile bulk copies and never used
    CK(cudaMemsetAsync(s.row_ptr.get(), 0, (n_rows + 1 + kRowSlack) * sizeof(uint64_t), st));
    CK(cudaMemsetAsync(s.target.get(), 0, (n_rows + kRowSlack) * sizeof(float), st));
    CK(cudaMemsetAsync(s.col.get(), 0, (nnz + kEntrySlack) * sizeof(uint32_t), st));
    CK(cudaMemsetAsync(s.val.get(), 0, (nnz + kEntrySlack) * sizeof(float), st));
    s.cap_rows = n_rows;
    s.cap_nnz = nnz;
  }
  CK(cudaMemsetAsync(s.d_flag.get(), 0, 16 * sizeof(unsigned int), st));  // the upload's verdicts start at 0
  s.present = false;
  s.links_ready = false;
  s.upload_gen = ++c->upload_counter;
  s.hogwild_epochs = 0;
  s.n_rows = n_rows;
  s.nnz = nnz;
  return 0;
}

// Inspection runs on the device: offsets monotone and consistent, longest row, tile
// spans, largest column id (the reference asserts id < num_attribute per access,
// fm_model.h:112), and the per-feature occurrence counts used by the HOGWILD damping.
// Leaves the results in the slot's pinned flag mirror (zeroed by upload_begin; words 0-9, and word 10
// for .x blocks); upload_finish() collects them.
int upload_inspect(fmb200_ctx* c, int slot, cudaStream_t st) {
  DataSlot& s = c->slots[slot];
  unsigned int* flag = s.d_flag.get();
  CK(launch_csr_inspect(c, st, s.row_ptr.get(), s.n_rows, s.nnz, flag));
  CK(launch_feature_counts(c, st, s.col.get(), s.nnz, s.feat_cnt.get(), flag + 8, flag + 9));
  CK(cudaMemcpyAsync(s.h_flag.get(), flag, 16 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(s.ready.get(), st));
  s.pending = true;
  return 0;
}

// Enqueue the copies + the device-side inspection of one SoA data set on `st`.
int upload_enqueue(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, const uint64_t* row_ptr,
                   const uint32_t* col, const float* val, const float* target, cudaStream_t st) {
  if (upload_begin(c, slot, n_rows, nnz, st)) return 1;
  DataSlot& s = c->slots[slot];
  CK(cudaMemcpyAsync(s.row_ptr.get(), row_ptr, (n_rows + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.target.get(), target, n_rows * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.col.get(), col, nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.val.get(), val, nnz * sizeof(float), cudaMemcpyHostToDevice, st));
  return upload_inspect(c, slot, st);
}

// One-hot rows of fixed width z: ids [n_rows*z] and targets cross PCIe; row offsets and the
// all-ones values are written by a kernel (fm_upload.cu).
int upload_onehot_enqueue(fmb200_ctx* c, int slot, uint64_t n_rows, uint32_t z, const uint32_t* ids,
                          const float* target, cudaStream_t st) {
  const uint64_t nnz = n_rows * z;
  if (upload_begin(c, slot, n_rows, nnz, st)) return 1;
  DataSlot& s = c->slots[slot];
  CK(cudaMemcpyAsync(s.target.get(), target, n_rows * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.col.get(), ids, nnz * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(launch_onehot_fill(c, st, n_rows, z, s.row_ptr.get(), s.val.get()));
  return upload_inspect(c, slot, st);
}

// The one host sync of an upload: wait for the slot's event and read the verdict.  deal: build the
// row-lane epoch's dealt copy now (a synchronous upload: a data set loaded to be trained on; one streamed
// in asynchronously is dealt at its second epoch, see launch_rowlane).
int upload_finish(fmb200_ctx* c, int slot, bool deal = false) {
  DataSlot& s = c->slots[slot];
  if (!s.pending) return 0;
  CK(cudaEventSynchronize(s.ready.get()));
  s.pending = false;
  const unsigned int* h = s.h_flag.get();
  if (h[10]) return fail("row %llu of the .x block: its header word is not row_size[%llu]",
                         (unsigned long long)(s.n_rows - h[10]), (unsigned long long)(s.n_rows - h[10]));
  if (h[0] & 1u) return fail("row_ptr[0] must be 0");
  if (h[0] & 2u) return fail("row_ptr is not monotone");
  if (h[0] & 4u) return fail("row_ptr[n_rows] != nnz");
  if (h[0] & 8u) return fail("a row is longer than 2^32-1 entries");
  if (s.nnz > 0 && h[8] >= c->n)
    return fail("feature id %u out of range (num_attribute=%u)", h[8], c->n);
  s.max_row_nnz = h[1];
  for (int i = 0; i < 5; i++) s.tile_span[i] = h[2 + i];
  s.max_feat_cnt = h[9];
  s.present = true;
  if (deal) CK(prepare_rowlane_deal(c, s));
  return 0;
}

int upload_common(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, const uint64_t* row_ptr,
                  const uint32_t* col, const float* val, const float* target) {
  if (upload_enqueue(c, slot, n_rows, nnz, row_ptr, col, val, target, c->stream)) return 1;
  return upload_finish(c, slot, true);
}

int need_slot(fmb200_ctx* c, int slot) {
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (c->slots[slot].pending && upload_finish(c, slot)) return 1;
  if (!c->slots[slot].present) return fail("slot %d holds no data", slot);
  return 0;
}

// the fp64 learners need an fp64 mode (INORDER or ORDERED) to be live; `what` says which needs it
int need_fp64(const fmb200_ctx* c, const char* what) {
  if (c->mode == FMB200_MODE_HOGWILD) return fail("%s", what);
  return 0;
}

// body() between the context's two events; *device_seconds (may be null) := the time between them
template <class F>
int timed(fmb200_ctx* c, double* device_seconds, F&& body) {
  CK(cudaEventRecord(c->ev0.get(), c->stream));
  if (body()) return 1;
  CK(cudaEventRecord(c->ev1.get(), c->stream));
  CK(cudaStreamSynchronize(c->stream));
  if (device_seconds) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev0.get(), c->ev1.get()));
    *device_seconds = (double)ms * 1e-3;
  }
  return 0;
}

}  // namespace

constexpr int kMaxPhaseSlots = 16;

cudaError_t PhaseTimers::start(int n_slots, cudaStream_t st) {
  if (n_slots > kMaxPhaseSlots) return cudaErrorInvalidValue;
  n = n_slots;
  const cudaError_t e = alloc(slots, (uint64_t)n);
  return e != cudaSuccess ? e : cudaMemsetAsync(slots.get(), 0, n * sizeof(unsigned long long), st);
}

cudaError_t PhaseTimers::print(cudaStream_t st, const char* const* names, double per, int decimals, bool skip_zero,
                               const char* head, ...) {
  unsigned long long h[kMaxPhaseSlots];
  cudaError_t e = cudaMemcpyAsync(h, slots.get(), n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return e;
  va_list ap;
  va_start(ap, head);
  vfprintf(stderr, head, ap);
  va_end(ap);
  for (int i = 0; i < n; i++)
    if (h[i] || !skip_zero) fprintf(stderr, " %s=%.*f", names[i], decimals, (double)h[i] / per);
  fprintf(stderr, "\n");
  return cudaSuccess;
}

// Everything of fmb200_create that can fail after the context object exists; the caller
// destroys the partially built context on a non-zero return.
static int create_resources(fmb200_ctx* c, int device, const cudaDeviceProp& prop, uint32_t n_attr,
                            int num_factor, int use_w0, int use_w) {
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  c->n = n_attr;
  c->k = num_factor;
  c->kp = (num_factor + 3) & ~3;
  c->k0 = use_w0 != 0;
  c->k1 = use_w != 0;
  CK(cudaSetDevice(device));
  CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CK(event_create(c->ev0, cudaEventDefault));
  CK(event_create(c->ev1, cudaEventDefault));
  c->p32.ws = (n_attr <= 131072u) ? 8 : 1;
  // w and V start on 128-byte lines (Params32): a k = 8 factor row is then exactly one 32-byte sector
  const uint64_t w_floats = ((uint64_t)n_attr * c->p32.ws + Params32::align - 1) & ~(Params32::align - 1);
  c->p32.off_w = Params32::align;
  c->p32.off_v = c->p32.off_w + w_floats;
  c->p32.n_floats = c->p32.off_v + (uint64_t)n_attr * c->kp;
  c->p64.off_v = Params64::off_w + (((uint64_t)n_attr + 1) & ~1ull);
  c->p64.n_doubles = c->p64.off_v + (uint64_t)n_attr * num_factor + 2;
  c->comm = CommLayout(c->p32.n_floats, n_attr);
  CK(alloc(c->comm_base, c->comm.total_bytes()));
  CK(cudaMemsetAsync(c->comm_base.get(), 0, c->comm.total_bytes(), c->stream));
  c->p32.base = c->comm.buf(c->comm_base.get(), 0);
  c->peer_base[0] = c->comm_base.get();
  CK(alloc(c->p64_buf, c->p64.n_doubles));
  c->p64.base = c->p64_buf.get();
  CK(cudaMemsetAsync(c->p32.base, 0, c->p32.n_floats * sizeof(float), c->stream));
  CK(cudaMemsetAsync(c->p64.base, 0, c->p64.n_doubles * sizeof(double), c->stream));
  CK(alloc(c->d_sched, 2));
  CK(cudaMemsetAsync(c->d_sched.get(), 0, 2 * sizeof(unsigned int), c->stream));
  CK(alloc(c->d_gbar, 1));
  CK(cudaMemsetAsync(c->d_gbar.get(), 0, sizeof(unsigned int), c->stream));
  CK(alloc(c->d_flag, 16));
  CK(host_alloc(c->h_flag, 16));
  {
    const size_t need = std::max(c->p32.n_floats * sizeof(float), c->p64.n_doubles * sizeof(double));
    if (need <= (64u << 20)) CK(host_alloc(c->h_stage, need));
  }
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

extern "C" {

const char* fmb200_last_error(void) { return g_err; }

int fmb200_create(fmb200_ctx** out, int device, uint32_t n_attr, int num_factor, int use_w0,
                  int use_w) {
  if (out == nullptr) return fail("null out pointer");
  *out = nullptr;
  if (num_factor < 0) return fail("num_factor must be >= 0");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail("no CUDA device available (%s): libfmb200 has no CPU path",
                e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  if (device < 0 || device >= count) return fail("device %d out of range (count %d)", device, count);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail("device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major,
                prop.minor);
  fmb200_ctx* c = new (std::nothrow) fmb200_ctx();
  if (!c) return fail("out of host memory");
  if (create_resources(c, device, prop, n_attr, num_factor, use_w0, use_w)) {
    fmb200_destroy(c);  // releases whatever was allocated; g_err keeps the cause
    return 1;
  }
  *out = c;
  return 0;
}

void fmb200_destroy(fmb200_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (int q = 0; q < FMB200_MAX_PEERS; q++)
    if (c->peer_ipc[q] && c->peer_base[q]) cudaIpcCloseMemHandle(c->peer_base[q]);
  cudaStream_t stream = c->stream, copy_stream = c->copy_stream;
  delete c;  // the owning handles release every buffer and event
  if (copy_stream) cudaStreamDestroy(copy_stream);
  if (stream) cudaStreamDestroy(stream);
}

int fmb200_set_hparams(fmb200_ctx* c, int task, double learn_rate, double reg0, double regw,
                       double regv, double min_target, double max_target) {
  NEED_CTX(c);
  if (task != FMB200_TASK_REGRESSION && task != FMB200_TASK_CLASSIFICATION)
    return fail("unknown task");  // fm_learn.h:99-101 throws "unknown task"
  c->hp.task = task;
  c->hp.lr = learn_rate;
  c->hp.reg0 = reg0;
  c->hp.regw = regw;
  c->hp.regv = regv;
  c->hp.min_target = min_target;
  c->hp.max_target = max_target;
  return 0;
}

int fmb200_set_mode(fmb200_ctx* c, int mode) {
  NEED_CTX(c);
  if (mode != FMB200_MODE_INORDER && mode != FMB200_MODE_HOGWILD && mode != FMB200_MODE_ORDERED)
    return fail("unknown mode %d", mode);
  if (mode == c->mode) return 0;
  if (bind(c)) return 1;
  // carry the live state into the representation of the new mode (INORDER and ORDERED share
  // the fp64 state)
  const bool was64 = c->mode != FMB200_MODE_HOGWILD, is64 = mode != FMB200_MODE_HOGWILD;
  if (is64 && c->k > 256) return fail("num_factor > 256 is not supported in the fp64 modes");
  if (was64 && !is64) {
    CK(launch_p64_to_p32(c));
  } else if (!was64 && is64) {
    CK(launch_p32_to_p64(c));
  }
  CK(cudaStreamSynchronize(c->stream));
  c->mode = mode;
  c->peer_base_valid = false;
  return 0;
}

int fmb200_upload_data(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz,
                       const uint64_t* row_ptr, const uint32_t* col, const float* val,
                       const float* target) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (!row_ptr || (n_rows && !target) || (nnz && (!col || !val))) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  if (bind(c)) return 1;
  return upload_common(c, slot, n_rows, nnz, row_ptr, col, val, target);
}

int fmb200_upload_data_async(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz,
                             const uint64_t* row_ptr, const uint32_t* col, const float* val,
                             const float* target) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (!row_ptr || (n_rows && !target) || (nnz && (!col || !val))) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  if (bind(c)) return 1;
  if (c->copy_stream == nullptr) CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  return upload_enqueue(c, slot, n_rows, nnz, row_ptr, col, val, target, c->copy_stream);
}

// reference layout, util/fmatrix.h:34-42
struct AosEntry {
  uint32_t id;
  float value;
};
struct AosRow {
  const AosEntry* data;
  uint32_t size;
};
static_assert(sizeof(AosRow) == 16 && sizeof(AosEntry) == 8, "LP64 layout of sparse_row/sparse_entry");

// rows scattered over the heap: gather them on the host (slow path)
static int upload_aos_host_gather(fmb200_ctx* c, int slot, uint64_t n_rows, const AosRow* r,
                                  const float* target) {
  return guarded([&]() -> int {
    std::vector<uint64_t> rp(n_rows + 1);
    rp[0] = 0;
    for (uint64_t i = 0; i < n_rows; i++) rp[i + 1] = rp[i] + r[i].size;
    const uint64_t nnz = rp[n_rows];
    std::vector<uint32_t> col(nnz ? nnz : 1);
    std::vector<float> val(nnz ? nnz : 1);
    for (uint64_t i = 0; i < n_rows; i++) {
      const AosEntry* e = r[i].data;
      uint64_t o = rp[i];
      for (uint32_t j = 0; j < r[i].size; j++) {
        col[o + j] = e[j].id;
        val[o + j] = e[j].value;
      }
    }
    return upload_common(c, slot, n_rows, nnz, rp.data(), col.data(), val.data(), target);
  });
}

int fmb200_upload_data_aos(fmb200_ctx* c, int slot, uint64_t n_rows, const void* rows,
                           const float* target) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (n_rows && (!rows || !target)) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  if (bind(c)) return 1;
  const AosRow* r = static_cast<const AosRow*>(rows);
  // The reference keeps all entries in ONE block (Data.h:238,260).  The row array crosses PCIe
  // as it is; the device scans the sizes into row offsets and checks that every row pointer is
  // where a contiguous block puts it.  Only then is the block itself read (8 B per entry, one
  // copy) and split into ids / values on the device.
  uint64_t first = 0;
  while (first < n_rows && r[first].size == 0) first++;
  if (first == n_rows) {  // no entries at all
    std::vector<uint64_t> rp;
    try {
      rp.assign(n_rows + 1, 0);
    } catch (const std::bad_alloc&) {
      return fail("out of host memory");
    }
    uint32_t dc = 0;
    float dv = 0.f;
    return upload_common(c, slot, n_rows, 0, rp.data(), &dc, &dv, target);
  }
  const unsigned long long base = (unsigned long long)(uintptr_t)r[first].data;
  cudaStream_t st = c->stream;
  // temporaries of the upload, released on return
  DevPtr<AosRow> d_rows;
  DevPtr<uint64_t> d_rp;
  DevPtr<unsigned long long> d_scr;
  DevPtr<AosEntry> d_ent;
  unsigned int* flag = c->d_flag.get();
  CK(alloc(d_rows, n_rows));
  CK(alloc(d_rp, n_rows + 1));
  CK(alloc(d_scr, aos_scan_tiles(n_rows) + 1));
  CK(cudaMemsetAsync(flag, 0, 16 * sizeof(unsigned int), st));
  CK(cudaMemcpyAsync(d_rows.get(), r, n_rows * sizeof(AosRow), cudaMemcpyHostToDevice, st));
  CK(launch_aos_to_csr(c, st, d_rows.get(), nullptr, n_rows, 0, base, d_scr.get(), d_rp.get(), nullptr, nullptr, flag));
  uint64_t nnz = 0;
  CK(cudaMemcpyAsync(c->h_flag.get(), flag, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(&nnz, d_rp.get() + n_rows, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (c->h_flag.get()[0] != 0) return upload_aos_host_gather(c, slot, n_rows, r, target);
  if (upload_begin(c, slot, n_rows, nnz, st)) return 1;
  DataSlot& s = c->slots[slot];
  CK(alloc(d_ent, nnz));
  CK(cudaMemcpyAsync(d_ent.get(), r[first].data, nnz * sizeof(AosEntry), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.row_ptr.get(), d_rp.get(), (n_rows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
  CK(cudaMemcpyAsync(s.target.get(), target, n_rows * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(launch_aos_split(c, st, d_ent.get(), nnz, s.col.get(), s.val.get()));
  if (upload_inspect(c, slot, st)) return 1;
  return upload_finish(c, slot, true);  // syncs: the temporaries may be released
}

int fmb200_upload_onehot(fmb200_ctx* c, int slot, uint64_t n_rows, uint32_t nnz_per_row,
                         const uint32_t* ids, const float* target) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (n_rows && (!target || (nnz_per_row && !ids))) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  if (bind(c)) return 1;
  if (upload_onehot_enqueue(c, slot, n_rows, nnz_per_row, ids, target, c->stream)) return 1;
  return upload_finish(c, slot, true);
}

int fmb200_upload_onehot_async(fmb200_ctx* c, int slot, uint64_t n_rows, uint32_t nnz_per_row,
                               const uint32_t* ids, const float* target) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (n_rows && (!target || (nnz_per_row && !ids))) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  if (bind(c)) return 1;
  if (c->copy_stream == nullptr) CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  return upload_onehot_enqueue(c, slot, n_rows, nnz_per_row, ids, target, c->copy_stream);
}

// n_rows rows of a .x file as it stores them (words: per row {size; size x {id, value}}): the words, the
// sizes and the targets cross PCIe; row offsets, the header check and the id / value split run on the device.
static int upload_xblock_enqueue(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, const void* words,
                                 const uint32_t* row_size, const float* target, cudaStream_t st) {
  if (upload_begin(c, slot, n_rows, nnz, st)) return 1;
  DataSlot& s = c->slots[slot];
  const uint64_t n_words = n_rows + 2 * nnz;
  CK(grow(s.x_words, s.x_words_cap, n_words ? n_words : 1));
  CK(grow(s.x_row_size, s.x_row_size_cap, n_rows ? n_rows : 1));
  CK(grow(s.x_scan, s.x_scan_cap, aos_scan_tiles(n_rows) + 1));
  CK(cudaMemcpyAsync(s.x_words.get(), words, n_words * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.x_row_size.get(), row_size, n_rows * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.target.get(), target, n_rows * sizeof(float), cudaMemcpyHostToDevice, st));
  CK(launch_xblock_to_csr(c, st, s.x_words.get(), s.x_row_size.get(), n_rows, nnz, s.x_scan.get(), s.row_ptr.get(),
                          s.col.get(), s.val.get(), s.d_flag.get() + 10));
  return upload_inspect(c, slot, st);
}

static int xblock_args(fmb200_ctx* c, int slot, uint64_t n_rows, const void* words, const uint32_t* row_size,
                       const float* target) {
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (n_rows && (!words || !row_size || !target)) return fail("null data pointer");
  if (n_rows > 0xffffffffull) return fail("row count exceeds the reference's uint range");
  return bind(c);
}

int fmb200_upload_xblock(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, const void* words,
                         const uint32_t* row_size, const float* target) {
  NEED_CTX(c);
  if (xblock_args(c, slot, n_rows, words, row_size, target)) return 1;
  if (upload_xblock_enqueue(c, slot, n_rows, nnz, words, row_size, target, c->stream)) return 1;
  return upload_finish(c, slot, true);
}

int fmb200_upload_xblock_async(fmb200_ctx* c, int slot, uint64_t n_rows, uint64_t nnz, const void* words,
                               const uint32_t* row_size, const float* target) {
  NEED_CTX(c);
  if (xblock_args(c, slot, n_rows, words, row_size, target)) return 1;
  if (c->copy_stream == nullptr) CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  return upload_xblock_enqueue(c, slot, n_rows, nnz, words, row_size, target, c->copy_stream);
}

}  // extern "C"

namespace fmb {

int upload_xt_enqueue(fmb200_ctx* c, int slot, uint64_t n_cols, uint64_t nnz, const void* words,
                      const uint32_t* col_size, cudaStream_t st) {
  if (upload_begin(c, slot, n_cols, nnz, st)) return 1;
  DataSlot& s = c->slots[slot];
  const uint64_t n_words = n_cols + 2 * nnz;
  CK(grow(s.x_words, s.x_words_cap, n_words ? n_words : 1));
  CK(grow(s.x_row_size, s.x_row_size_cap, n_cols ? n_cols : 1));
  CK(grow(s.x_scan, s.x_scan_cap, aos_scan_tiles(n_cols) + 1));
  CK(cudaMemcpyAsync(s.x_words.get(), words, n_words * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s.x_row_size.get(), col_size, n_cols * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  CK(launch_xblock_to_csr(c, st, s.x_words.get(), s.x_row_size.get(), n_cols, nnz, s.x_scan.get(), s.row_ptr.get(),
                          s.col.get(), s.val.get(), s.d_flag.get() + 10));
  CK(launch_max_id(c, st, s.col.get(), nnz, s.d_flag.get() + 8));
  CK(cudaMemcpyAsync(s.h_flag.get(), s.d_flag.get(), 16 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(s.ready.get(), st));
  s.pending = true;
  return 0;
}

int upload_xt_finish(fmb200_ctx* c, int slot, uint64_t first_col, uint64_t n_cases) {
  DataSlot& s = c->slots[slot];
  if (!s.pending) return 0;
  CK(cudaEventSynchronize(s.ready.get()));
  s.pending = false;
  const unsigned int* h = s.h_flag.get();
  if (h[10]) return fail("column %llu of the .xt: its header word is not its size",
                         (unsigned long long)(first_col + s.n_rows - h[10]));
  if (s.nnz > 0 && h[8] >= n_cases)
    return fail("case id %u in the .xt block from column %llu is out of range (%llu cases)", h[8],
                (unsigned long long)first_col, (unsigned long long)n_cases);
  s.present = true;
  return 0;
}

}  // namespace fmb

extern "C" {

int fmb200_host_alloc(void** out, uint64_t bytes) {
  if (!out) return fail("null out pointer");
  *out = nullptr;
  CK(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return 0;
}

int fmb200_host_free(void* p) {
  if (p) CK(cudaFreeHost(p));
  return 0;
}

int fmb200_free_data(fmb200_ctx* c, int slot) {
  NEED_CTX(c);
  if (slot < 0 || slot >= FMB200_MAX_SLOTS) return fail("slot %d out of range", slot);
  if (bind(c)) return 1;
  CK(cudaStreamSynchronize(c->stream));
  if (c->slots[slot].pending) CK(cudaEventSynchronize(c->slots[slot].ready.get()));
  c->slots[slot] = DataSlot();
  return 0;
}

int fmb200_set_params(fmb200_ctx* c, double w0, const double* w, const double* v) {
  NEED_CTX(c);
  if ((c->n && !w) || ((uint64_t)c->n * c->k && !v)) return fail("null parameter pointer");
  if (bind(c)) return 1;
  return guarded([&]() -> int {
  const uint32_t n = c->n;
    const int k = c->k, kp = c->kp;
    // fp64 image: [w0 | w | V attribute-major]
    std::vector<double> h64(c->p64.n_doubles);
    h64[0] = w0;
    for (uint32_t i = 0; i < n; i++) h64[Params64::off_w + i] = w[i];
    double* hv = h64.data() + c->p64.off_v;
    for (int f = 0; f < k; f++)
      for (uint32_t i = 0; i < n; i++) hv[(size_t)i * k + f] = v[(size_t)f * n + i];
    // fp32 packed image
    std::vector<float> h32(c->p32.n_floats, 0.f);
    h32[0] = (float)w0;
    for (uint32_t i = 0; i < n; i++) h32[c->p32.off_w + (size_t)i * c->p32.ws] = (float)w[i];
    float* hv32 = h32.data() + c->p32.off_v;
    for (int f = 0; f < k; f++)
      for (uint32_t i = 0; i < n; i++) hv32[(size_t)i * kp + f] = (float)v[(size_t)f * n + i];
    CK(cudaMemcpyAsync(c->p64.base, h64.data(), h64.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->p32.base, h32.data(), h32.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    CK(clear_acc_flag(c));
    CK(cudaStreamSynchronize(c->stream));
    c->peer_base_valid = false;
    c->hogwild_fresh = true;
    return 0;
  });
}

int fmb200_get_params(fmb200_ctx* c, double* w0, double* w, double* v) {
  NEED_CTX(c);
  if (!w0 || (c->n && !w) || ((uint64_t)c->n * c->k && !v)) return fail("null parameter pointer");
  if (bind(c)) return 1;
  return guarded([&]() -> int {
  const uint32_t n = c->n;
    const int k = c->k, kp = c->kp;
    if (c->mode != FMB200_MODE_HOGWILD) {
      std::vector<double> pageable;
      double* h = reinterpret_cast<double*>(c->h_stage.get());  // pinned staging for small models
      if (h == nullptr) {
        pageable.resize(c->p64.n_doubles);
        h = pageable.data();
      }
      CK(cudaMemcpyAsync(h, c->p64.base, c->p64.n_doubles * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
      CK(cudaStreamSynchronize(c->stream));
      *w0 = h[0];
      for (uint32_t i = 0; i < n; i++) w[i] = h[Params64::off_w + i];
      const double* hv = h + c->p64.off_v;
      for (int f = 0; f < k; f++)
        for (uint32_t i = 0; i < n; i++) v[(size_t)f * n + i] = hv[(size_t)i * k + f];
    } else {
      std::vector<float> pageable;
      float* h = reinterpret_cast<float*>(c->h_stage.get());
      if (h == nullptr) {
        pageable.resize(c->p32.n_floats);
        h = pageable.data();
      }
      CK(cudaMemcpyAsync(h, c->p32.base, c->p32.n_floats * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
      CK(cudaStreamSynchronize(c->stream));
      *w0 = h[0];
      for (uint32_t i = 0; i < n; i++) w[i] = h[c->p32.off_w + (size_t)i * c->p32.ws];
      const float* hv = h + c->p32.off_v;
      for (uint32_t i = 0; i < n; i++)
        for (int f = 0; f < k; f++) v[(size_t)f * n + i] = hv[(size_t)i * kp + f];
    }
    return 0;
  });
}

int fmb200_sgd_epoch_async(fmb200_ctx* c, int slot) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  DataSlot& d = c->slots[slot];
  if (c->mode == FMB200_MODE_ORDERED) {
    bool handled = false;
    CK(launch_sgd_ordered(c, d, &handled));
    // shapes the ring cannot hold run row-at-a-time: the same order, just slower
    if (!handled) CK(launch_sgd_inorder(c, d));
  } else if (c->mode == FMB200_MODE_INORDER) {
    CK(launch_sgd_inorder(c, d));
  } else {
    if (c->kp > 128) return fail("num_factor > 128 is not supported in HOGWILD mode");
    CK(peer_before_epoch(c, d));  // multi-GPU: theta0 + shard counts for the mean-field combine
    CK(launch_sgd_hogwild(c, d));
  }
  return 0;
}

int fmb200_sync(fmb200_ctx* c) {
  NEED_CTX(c);
  if (bind(c)) return 1;
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_sgd_epoch(fmb200_ctx* c, int slot, double* device_seconds) {
  NEED_CTX(c);
  if (bind(c)) return 1;
  return timed(c, device_seconds, [&] { return fmb200_sgd_epoch_async(c, slot); });
}

int fmb200_evaluate(fmb200_ctx* c, int slot, double* sum_sq_err, double* sum_abs_err,
                    uint64_t* n_correct) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  const DataSlot& d = c->slots[slot];
  double sq = 0, ab = 0, ok = 0;
  if (d.n_rows > 0) {
    const int nb = grid_for(c, d.n_rows);
    CK(grow(c->d_partials, c->n_partials, 3 * (uint64_t)nb));
    if (c->mode != FMB200_MODE_HOGWILD && c->hp.task == FMB200_TASK_REGRESSION) {
      // fp64 modes: the reference sums err*err and |err| left to right over the rows
      // (fm_learn.h:136-146); a tree reduction may differ in the last ulps and flip a printed
      // digit.  The kernel writes the per-row error, the host adds them in row order.
      CK(grow(c->d_pred, c->pred_cap, d.n_rows));
      CK(launch_predict64(c, d, 2, c->d_pred.get(), nullptr, nb));
      std::vector<double> err;
      try {
        err.resize(d.n_rows);
      } catch (const std::bad_alloc&) {
        return fail("out of host memory");
      }
      CK(cudaMemcpyAsync(err.data(), c->d_pred.get(), d.n_rows * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
      CK(cudaStreamSynchronize(c->stream));
      for (uint64_t i = 0; i < d.n_rows; i++) {
        sq += err[i] * err[i];
        ab += std::abs(err[i]);
      }
    } else {
      if (c->mode != FMB200_MODE_HOGWILD) {
        CK(launch_predict64(c, d, 0, nullptr, c->d_partials.get(), nb));
      } else {
        CK(launch_predict32(c, d, 0, nullptr, c->d_partials.get(), nb));
      }
      std::vector<double> h;
      try {
        h.resize(3 * (size_t)nb);
      } catch (const std::bad_alloc&) {
        return fail("out of host memory");
      }
      CK(cudaMemcpyAsync(h.data(), c->d_partials.get(), h.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
      CK(cudaStreamSynchronize(c->stream));
      for (int b = 0; b < nb; b++) {  // fixed order: deterministic result
        sq += h[3 * b + 0];
        ab += h[3 * b + 1];
        ok += h[3 * b + 2];
      }
    }
  }
  if (sum_sq_err) *sum_sq_err = sq;
  if (sum_abs_err) *sum_abs_err = ab;
  if (n_correct) *n_correct = (uint64_t)llround(ok);
  return 0;
}

int fmb200_predict(fmb200_ctx* c, int slot, int transform, double* out) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  const DataSlot& d = c->slots[slot];
  if (d.n_rows == 0) return 0;
  if (!out) return fail("null output pointer");
  CK(grow(c->d_pred, c->pred_cap, d.n_rows));
  const int nb = grid_for(c, d.n_rows);
  if (c->mode != FMB200_MODE_HOGWILD) {
    CK(launch_predict64(c, d, transform, c->d_pred.get(), nullptr, nb));
  } else {
    CK(launch_predict32(c, d, transform, c->d_pred.get(), nullptr, nb));
  }
  CK(cudaMemcpyAsync(out, c->d_pred.get(), d.n_rows * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_sgda_begin(fmb200_ctx* c, uint32_t n_groups, const uint32_t* attr_group) {
  NEED_CTX(c);
  if (bind(c)) return 1;
  const bool hogwild = c->mode == FMB200_MODE_HOGWILD;
  if (n_groups == 0) return fail("n_groups must be in [1,1024]");
  if (hogwild && c->k > 128) return fail("SGDA in HOGWILD mode supports num_factor <= 128 (got %d)", c->k);
  // before the group cap: at num_factor = 7 both allow 1024 groups, and the refusal of 1025 names both
  if (hogwild && (uint64_t)n_groups * (c->k + 1) > kSgdaMaxTerms)
    return fail("SGDA in HOGWILD mode with %u groups at num_factor = %d keeps %llu lambda terms per validation row "
                "(groups * (num_factor + 1)); at most %llu: use at most %llu groups",
                n_groups, c->k, (unsigned long long)n_groups * (c->k + 1), (unsigned long long)kSgdaMaxTerms,
                (unsigned long long)std::min<uint64_t>(1024, kSgdaMaxTerms / (c->k + 1)));
  if (n_groups > 1024) return fail("n_groups must be in [1,1024]");
  if (n_groups > 1 && !attr_group) return fail("attr_group is required for more than one group");
  if (!hogwild && sgda_smem_bytes(n_groups, c->k) > (size_t)c->max_smem_optin)
    return fail("SGDA with %u groups at num_factor = %d needs %zu bytes of shared memory per block (8 * groups * "
                "(2 + 3 * num_factor)); this device allows %d: use at most %zu groups",
                n_groups, c->k, sgda_smem_bytes(n_groups, c->k), c->max_smem_optin,
                (size_t)c->max_smem_optin / sgda_smem_bytes(1, c->k));
  if (attr_group)
    for (uint32_t i = 0; i < c->n; i++)
      if (attr_group[i] >= n_groups) return fail("attr_group[%u] = %u >= n_groups", i, attr_group[i]);
  const size_t n1 = c->n ? c->n : 1, nk = (size_t)c->n * c->k ? (size_t)c->n * c->k : 1;
  const size_t gk = (size_t)n_groups * (c->k ? c->k : 1);
  if (!c->sgda_grad_w) {
    CK(alloc(c->sgda_grad_w, n1));
    CK(alloc(c->sgda_grad_v, nk));
    CK(alloc(c->sgda_group, n1));
    CK(alloc(c->sgda_moments, 1 + (size_t)c->k));
  }
  c->sgda_moments_ready = false;
  if (c->sgda_groups != n_groups) {
    c->sgda_groups = 0;
    CK(alloc(c->sgda_reg_w, n_groups));
    CK(alloc(c->sgda_reg_v, gk));
    c->sgda_groups = n_groups;
  }
  // init(): grad_w = grad_v = 0 (:73-74); learn(): w = 0, reg_w = reg_v = 0 (:283-291)
  CK(cudaMemsetAsync(c->sgda_grad_w.get(), 0, n1 * sizeof(double), c->stream));
  CK(cudaMemsetAsync(c->sgda_grad_v.get(), 0, nk * sizeof(double), c->stream));
  CK(cudaMemsetAsync(c->sgda_reg_w.get(), 0, n_groups * sizeof(double), c->stream));
  CK(cudaMemsetAsync(c->sgda_reg_v.get(), 0, gk * sizeof(double), c->stream));
  if (hogwild) {  // the fp32 stored gradients and their window sums, beside the packed state
    const uint64_t nf = c->p32.n_floats;
    if (!c->sgda_grad32) {
      CK(alloc(c->sgda_grad32, nf));
      CK(alloc(c->sgda_gacc, nf));
    }
    CK(cudaMemsetAsync(c->sgda_grad32.get(), 0, nf * sizeof(float), c->stream));
    CK(cudaMemsetAsync(c->sgda_gacc.get(), 0, nf * sizeof(unsigned long long), c->stream));
    CK(cudaMemsetAsync(c->p32.w(), 0, (size_t)c->n * c->p32.ws * sizeof(float), c->stream));
    CK(clear_acc_flag(c));
  } else {
    CK(cudaMemsetAsync(c->p64.w(), 0, n1 * sizeof(double), c->stream));
  }
  if (attr_group) CK(cudaMemcpyAsync(c->sgda_group.get(), attr_group, c->n * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
  else CK(cudaMemsetAsync(c->sgda_group.get(), 0, n1 * sizeof(uint32_t), c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // extern "C"

namespace {

// A data set of an SGDA epoch: resident in `slot`, or streamed from the .x blocks `src` through src->slot[0] and
// src->slot[1].  order: the blocks the epoch's launches read, in turn (a block read by consecutive launches once);
// order[j] passes through src->slot[j % 2], so the next block's copy overlaps the launches on this one.
struct SgdaSet {
  const char* name;
  int slot = -1;
  const fmb200_xt_blocks* src = nullptr;
  uint64_t rows = 0;
  std::vector<int64_t> order;
  size_t pos = 0;  // order[pos] is in use (once started)
  bool started = false;

  const uint32_t* lo() const { return src ? src->col_lo : nullptr; }
  uint64_t n_blocks() const { return src ? src->n_blocks : 0; }
  int slot_of(size_t j) const { return src->slot[j % 2]; }
  uint64_t row0() const { return started ? src->col_lo[order[pos]] : 0; }
};

// the checks of a streamed .x set: its block plan must cover its rows in order
int sgda_check_blocks(const SgdaSet& s) {
  const fmb200_xt_blocks& x = *s.src;
  if (x.n_blocks == 0 || !x.col_lo || !x.nnz || !x.fetch || !x.release)
    return fail("the %s .x blocks: no blocks or a null pointer", s.name);
  if (x.n_cases && !x.target) return fail("the %s .x blocks: null target", s.name);
  if (x.n_cases >= 0xffffffffull) return fail("the %s .x blocks: 2^32 rows and more are not supported", s.name);
  for (int i = 0; i < 2; i++)
    if (x.slot[i] < 0 || x.slot[i] >= FMB200_MAX_SLOTS) return fail("the %s .x blocks: slot out of range", s.name);
  if (x.slot[0] == x.slot[1]) return fail("the %s .x blocks: the two slots must differ", s.name);
  if (x.col_lo[0] != 0 || x.col_lo[x.n_blocks] != x.n_cases)
    return fail("the %s .x blocks: the rows must start at 0 and end at n_cases", s.name);
  for (uint64_t b = 0; b < x.n_blocks; b++) {
    if (x.col_lo[b + 1] < x.col_lo[b]) return fail("the %s .x blocks: row ranges out of order", s.name);
    if (x.nnz[b] >= 0xffffffffull) return fail("the %s .x blocks: a block of 2^32 entries and more", s.name);
  }
  return 0;
}

// Enqueue the copy and the decoding of order[j] into its slot on the copy stream
int sgda_enqueue(fmb200_ctx* c, SgdaSet& s, size_t j) {
  const uint64_t b = (uint64_t)s.order[j];
  const void* words = nullptr;
  const uint32_t* sizes = nullptr;
  if (s.src->fetch(s.src->user, b, &words, &sizes) != 0)
    return fail("fetching block %llu of the %s .x failed", (unsigned long long)b, s.name);
  const uint32_t lo = s.src->col_lo[b];
  return upload_xblock_enqueue(c, s.slot_of(j), s.src->col_lo[b + 1] - lo, s.src->nnz[b], words, sizes,
                               s.src->target + lo, c->copy_stream);
}

// Make block b the one the next launches read: wait for its copy, release it, and start the copy of the block
// after it into the other slot once the launches on that slot's block have run.
int sgda_advance(fmb200_ctx* c, SgdaSet& s, int64_t b) {
  if (b < 0 || (s.started && s.order[s.pos] == b)) return 0;
  const size_t j = s.started ? s.pos + 1 : 0;
  if (!s.started && sgda_enqueue(c, s, 0)) return 1;
  s.started = true;
  s.pos = j;
  if (upload_finish(c, s.slot_of(j))) {
    const std::string e = g_err;
    return fail("block %lld of the %s .x: %s", (long long)b, s.name, e.c_str());
  }
  s.src->release(s.src->user, (uint64_t)b);
  if (j + 1 < s.order.size()) {
    CK(cudaStreamSynchronize(c->stream));  // order[j - 1], whose slot the next block takes, is done with
    if (sgda_enqueue(c, s, j + 1)) return 1;
  }
  return 0;
}

// The epoch as sgda_plan cuts it, each streamed set's blocks fetched in the order its launches read them
int sgda_run(fmb200_ctx* c, SgdaSet& tr, SgdaSet& va, int lambda_steps) {
  const std::vector<SgdaLaunch> plan =
      sgda_plan(tr.rows, va.rows, lambda_steps != 0, tr.lo(), tr.n_blocks(), va.lo(), va.n_blocks());
  for (const SgdaLaunch& l : plan) {
    if (tr.src && l.train_block >= 0 && (tr.order.empty() || tr.order.back() != l.train_block))
      tr.order.push_back(l.train_block);
    if (va.src && l.val_block >= 0 && (va.order.empty() || va.order.back() != l.val_block))
      va.order.push_back(l.val_block);
  }
  for (const SgdaLaunch& l : plan) {
    if (sgda_advance(c, tr, l.train_block) || sgda_advance(c, va, l.val_block)) return 1;
    const DataSlot& ts = c->slots[tr.src ? tr.slot_of(tr.pos) : tr.slot];
    // a streamed validation set no launch has read yet stands in as the training block (no lambda-steps read it)
    const DataSlot& vs = va.src ? (va.started ? c->slots[va.slot_of(va.pos)] : ts) : c->slots[va.slot];
    CK(launch_sgda(c, l, lambda_steps, ts, tr.row0(), tr.rows, vs, va.row0(), va.rows));
  }
  return 0;
}

}  // namespace

extern "C" {

int fmb200_sgda_epoch_x(fmb200_ctx* c, int train_slot, const fmb200_xt_blocks* train, int val_slot,
                        const fmb200_xt_blocks* val, int lambda_steps, double* device_seconds) {
  NEED_CTX(c);
  if ((!train && need_slot(c, train_slot)) || (!val && need_slot(c, val_slot))) return 1;
  if (bind(c)) return 1;
  if (c->sgda_groups == 0) return fail("call fmb200_sgda_begin first");
  if (c->mode == FMB200_MODE_HOGWILD) {
    if (train || val)
      return fail("SGDA in HOGWILD mode takes resident data sets: streamed (.x block) SGDA runs in INORDER or "
                  "ORDERED mode");
    if (c->peer_world > 1) return fail("SGDA in HOGWILD mode runs on one GPU: this context has peers");
    if (!c->sgda_grad32) return fail("call fmb200_sgda_begin in HOGWILD mode first");
    return timed(c, device_seconds, [&]() -> int {
      CK(launch_sgda_hogwild(c, c->slots[train_slot], c->slots[val_slot], lambda_steps));
      c->sgda_moments_ready = true;
      return 0;
    });
  }
  SgdaSet tr{"training", train_slot, train}, va{"validation", val_slot, val};
  for (SgdaSet* s : {&tr, &va}) {
    if (!s->src) {
      s->rows = c->slots[s->slot].n_rows;
      continue;
    }
    if (c->peer_world > 1) return fail("a streamed SGDA epoch runs on one GPU: this context has peers");
    if (sgda_check_blocks(*s)) return 1;
    s->rows = s->src->n_cases;
  }
  {  // a streamed set's slots serve it alone
    std::vector<int> res, str;
    for (SgdaSet* s : {&tr, &va})
      if (s->src) str.insert(str.end(), {s->src->slot[0], s->src->slot[1]});
      else res.push_back(s->slot);
    for (size_t i = 0; i < str.size(); i++) {
      for (size_t j = 0; j < i; j++)
        if (str[i] == str[j]) return fail("a streamed set's slots must differ from every other slot in use");
      for (int r : res)
        if (str[i] == r) return fail("a streamed set's slots must differ from every other slot in use");
    }
  }
  if ((train || val) && c->copy_stream == nullptr) CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  return guarded([&]() -> int {
    return timed(c, device_seconds, [&]() -> int {
      if (sgda_run(c, tr, va, lambda_steps)) {
        if (train || val) cudaStreamSynchronize(c->copy_stream);  // no copy may still read a fetched block
        return 1;
      }
      c->sgda_moments_ready = true;
      return 0;
    });
  });
}

int fmb200_sgda_epoch(fmb200_ctx* c, int train_slot, int val_slot, int lambda_steps, double* device_seconds) {
  return fmb200_sgda_epoch_x(c, train_slot, nullptr, val_slot, nullptr, lambda_steps, device_seconds);
}

int fmb200_sgda_get_moments(fmb200_ctx* c, double* var_w, double* var_v) {
  NEED_CTX(c);
  if (bind(c)) return 1;
  if (c->sgda_groups == 0) return fail("call fmb200_sgda_begin first");
  if (!c->sgda_moments_ready) return fail("no SGDA epoch has run since fmb200_sgda_begin");
  if (var_w) CK(cudaMemcpyAsync(var_w, c->sgda_moments.get(), sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (var_v && c->k)
    CK(cudaMemcpyAsync(var_v, c->sgda_moments.get() + 1, (size_t)c->k * sizeof(double), cudaMemcpyDeviceToHost,
                       c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_sgda_get_reg(fmb200_ctx* c, double* reg_w, double* reg_v) {
  NEED_CTX(c);
  if (bind(c)) return 1;
  if (c->sgda_groups == 0) return fail("call fmb200_sgda_begin first");
  if (reg_w) CK(cudaMemcpyAsync(reg_w, c->sgda_reg_w.get(), c->sgda_groups * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (reg_v && c->k)
    CK(cudaMemcpyAsync(reg_v, c->sgda_reg_v.get(), (size_t)c->sgda_groups * c->k * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_mcmc_eterms(fmb200_ctx* c, int slot, double* e_out) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  if (need_fp64(c, "e-terms are computed from the fp64 state: set INORDER or ORDERED mode first")) return 1;
  const DataSlot& d = c->slots[slot];
  if (d.n_rows == 0) return 0;
  if (!e_out) return fail("null output pointer");
  CK(grow(c->d_pred, c->pred_cap, d.n_rows));
  CK(launch_mcmc_eterms(c, d, c->d_pred.get()));
  CK(cudaMemcpyAsync(e_out, c->d_pred.get(), d.n_rows * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

// The body of fmb200_mcmc_begin and fmb200_mcmc_begin_xt; fn names the entry point in messages
static int mcmc_begin_entry(const char* fn, fmb200_ctx* c, int train_slot, const fmb200_xt_blocks* train_xt,
                            int test_slot, const fmb200_xt_blocks* test_xt, int do_sample, int do_multilevel,
                            uint32_t n_groups, const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                            const double* w_lambda, const double* v_lambda) {
  NEED_CTX(c);
  struct DropRelations {  // relations set before apply to this call only, whichever way it ends
    fmb200_ctx* c;
    ~DropRelations() { c->mcmc_rel.clear(); }
  } drop{c};
  if ((!train_xt && need_slot(c, train_slot)) || (!test_xt && need_slot(c, test_slot))) return 1;
  if (bind(c)) return 1;
  if (need_fp64(c, "MCMC / ALS run on the fp64 state: set INORDER or ORDERED mode first")) return 1;
  if (!w_lambda || (!v_lambda && c->k > 0)) return fail("null w_lambda / v_lambda");
  if (c->peer_world > 1) return fail("MCMC / ALS run on one GPU: this context is attached to a multi-GPU peer world");
  if ((train_xt || test_xt) && c->copy_stream == nullptr)
    CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  return guarded([&]() {
    const std::string e = mcmc_begin(c, train_slot, test_slot, do_sample, do_multilevel, n_groups, attr_group,
                                      attr_per_group, reg0, w_lambda, v_lambda, train_xt, test_xt);
    if (!e.empty()) {
      c->mcmc.reset();
      return fail("%s: %s", fn, e.c_str());
    }
    return 0;
  });
}

int fmb200_mcmc_begin(fmb200_ctx* c, int train_slot, int test_slot, int do_sample, int do_multilevel,
                      uint32_t n_groups, const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                      const double* w_lambda, const double* v_lambda) {
  return mcmc_begin_entry("fmb200_mcmc_begin", c, train_slot, nullptr, test_slot, nullptr, do_sample, do_multilevel,
                          n_groups, attr_group, attr_per_group, reg0, w_lambda, v_lambda);
}

int fmb200_mcmc_set_relations(fmb200_ctx* c, int train_slot, int test_slot, uint32_t n_rel,
                              const fmb200_relation* rel) {
  NEED_CTX(c);
  c->mcmc_rel.clear();
  if (n_rel == 0) return 0;
  if (need_slot(c, train_slot) || need_slot(c, test_slot)) return 1;
  return guarded([&]() {
    std::vector<RelationHost> r;
    const std::string e = mcmc_check_relations(c, train_slot, test_slot, n_rel, rel, &r);
    if (!e.empty()) return fail("fmb200_mcmc_set_relations: %s", e.c_str());
    c->mcmc_rel = std::move(r);
    c->mcmc_rel_slot[0] = train_slot;
    c->mcmc_rel_slot[1] = test_slot;
    c->mcmc_rel_gen[0] = c->slots[train_slot].upload_gen;
    c->mcmc_rel_gen[1] = c->slots[test_slot].upload_gen;
    return 0;
  });
}

int fmb200_mcmc_begin_xt(fmb200_ctx* c, int train_slot, const fmb200_xt_blocks* train_xt, int test_slot,
                         const fmb200_xt_blocks* test_xt, int do_sample, int do_multilevel, uint32_t n_groups,
                         const uint32_t* attr_group, const uint32_t* attr_per_group, double reg0,
                         const double* w_lambda, const double* v_lambda) {
  NEED_CTX(c);
  if (!c->mcmc_rel.empty()) {
    c->mcmc_rel.clear();
    return fail("fmb200_mcmc_begin_xt: relations are not streamed: call fmb200_mcmc_begin for relational data");
  }
  return mcmc_begin_entry("fmb200_mcmc_begin_xt", c, train_slot, train_xt, test_slot, test_xt, do_sample, do_multilevel,
                          n_groups, attr_group, attr_per_group, reg0, w_lambda, v_lambda);
}

int fmb200_mcmc_iteration(fmb200_ctx* c, double* train_metric, uint32_t* counters) {
  NEED_CTX(c);
  if (!c->mcmc) return fail("call fmb200_mcmc_begin first");
  if (need_fp64(c, "MCMC / ALS run on the fp64 state: set INORDER or ORDERED mode first")) return 1;
  if (bind(c)) return 1;
  return guarded([&]() {
    double m = 0.0;
    const std::string e = mcmc_iteration(c, &m, counters);
    if (!e.empty()) return fail("fmb200_mcmc_iteration: %s", e.c_str());
    if (train_metric) *train_metric = m;
    return 0;
  });
}

int fmb200_mcmc_get_hyper(fmb200_ctx* c, double* alpha, double* w_mu, double* w_lambda, double* v_mu,
                          double* v_lambda) {
  NEED_CTX(c);
  if (!mcmc_get(c, alpha, w_mu, w_lambda, v_mu, v_lambda, nullptr, nullptr, nullptr, nullptr))
    return fail("call fmb200_mcmc_begin first");
  return 0;
}

int fmb200_mcmc_get_pred(fmb200_ctx* c, double* pred_this, double* pred_sum_all, double* pred_sum_all_but5) {
  NEED_CTX(c);
  if (!mcmc_get(c, nullptr, nullptr, nullptr, nullptr, nullptr, pred_this, pred_sum_all, pred_sum_all_but5, nullptr))
    return fail("call fmb200_mcmc_begin first");
  return 0;
}

int fmb200_mcmc_runs(fmb200_ctx* c, uint32_t* n_runs) {
  NEED_CTX(c);
  if (!mcmc_get(c, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, n_runs))
    return fail("call fmb200_mcmc_begin first");
  return 0;
}

int fmb200_params_device(fmb200_ctx* c, void** device_ptr, uint64_t* n_floats) {
  NEED_CTX(c);
  if (c->mode != FMB200_MODE_HOGWILD) return fail("packed fp32 state is live only in HOGWILD mode");
  if (device_ptr) *device_ptr = c->p32.base;
  if (n_floats) *n_floats = c->p32.n_floats;
  return 0;
}

int fmb200_params_layout(fmb200_ctx* c, uint64_t* off_w, int* ws, uint64_t* off_v, int* kp) {
  NEED_CTX(c);
  if (off_w) *off_w = c->p32.off_w;
  if (ws) *ws = c->p32.ws;
  if (off_v) *off_v = c->p32.off_v;
  if (kp) *kp = c->kp;
  return 0;
}

int fmb200_scale_params(fmb200_ctx* c, double factor) {
  NEED_CTX(c);
  if (c->mode != FMB200_MODE_HOGWILD) return fail("scale_params applies to the HOGWILD state");
  if (bind(c)) return 1;
  CK(launch_scale_p32(c, (float)factor));
  c->peer_base_valid = false;
  return 0;
}

int fmb200_peer_export(fmb200_ctx* c, void* handle) {
  NEED_CTX(c);
  if (!handle) return fail("null handle pointer");
  if (bind(c)) return 1;
  static_assert(sizeof(cudaIpcMemHandle_t) == FMB200_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, c->comm_base.get()));
  memcpy(handle, &h, sizeof(h));
  return 0;
}

static int peer_precheck(fmb200_ctx* c, int world, int rank) {
  if (world < 1 || world > FMB200_MAX_PEERS) return fail("world %d outside [1,%d]", world, FMB200_MAX_PEERS);
  if (rank < 0 || rank >= world) return fail("rank %d outside world %d", rank, world);
  if (c->peer_seq != 0 || c->peer_world != 1) return fail("peers are already attached");
  if (c->mode != FMB200_MODE_HOGWILD) return fail("peer averaging applies to the HOGWILD state");
  return 0;
}

int fmb200_peer_attach_ipc(fmb200_ctx* c, int world, int rank, const void* handles) {
  NEED_CTX(c);
  if (!handles) return fail("null handles");
  if (peer_precheck(c, world, rank)) return 1;
  if (bind(c)) return 1;
  const unsigned char* hb = static_cast<const unsigned char*>(handles);
  for (int q = 0; q < world; q++) {
    if (q == rank) {
      c->peer_base[q] = c->comm_base.get();
      continue;
    }
    cudaIpcMemHandle_t h;
    memcpy(&h, hb + (size_t)q * FMB200_IPC_HANDLE_BYTES, sizeof(h));
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer_base[q] = static_cast<unsigned char*>(p);
    c->peer_ipc[q] = true;
  }
  CK(peer_preload_kernels());
  c->peer_world = world;
  c->peer_rank = rank;
  return 0;
}

int fmb200_peer_attach_local(fmb200_ctx* c, int world, int rank, fmb200_ctx* const* all) {
  NEED_CTX(c);
  if (!all) return fail("null context list");
  if (peer_precheck(c, world, rank)) return 1;
  if (bind(c)) return 1;
  for (int q = 0; q < world; q++) {
    if (!all[q] || all[q]->p32.n_floats != c->p32.n_floats) return fail("peer %d has a different model shape", q);
    if (q != rank && all[q]->device != c->device) {
      int can = 0;
      CK(cudaDeviceCanAccessPeer(&can, c->device, all[q]->device));
      if (!can) return fail("device %d cannot access device %d", c->device, all[q]->device);
      cudaError_t e = cudaDeviceEnablePeerAccess(all[q]->device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
        return fail("cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
      (void)cudaGetLastError();
    }
    c->peer_base[q] = all[q]->comm_base.get();
  }
  CK(peer_preload_kernels());
  c->peer_world = world;
  c->peer_rank = rank;
  return 0;
}

int fmb200_allreduce_mean(fmb200_ctx* c) {
  NEED_CTX(c);
  if (c->mode != FMB200_MODE_HOGWILD) return fail("peer averaging applies to the HOGWILD state");
  if (c->peer_world <= 1) return 0;
  if (bind(c)) return 1;
  CK(launch_peer_mean(c));
  return 0;
}

int fmb200_allreduce_meanfield(fmb200_ctx* c) {
  NEED_CTX(c);
  if (c->mode != FMB200_MODE_HOGWILD) return fail("the peer exchange applies to the HOGWILD state");
  if (c->peer_world <= 1) return 0;
  if (!c->peer_base_valid) return fail("no epoch has run since the state was last set: nothing to combine");
  if (bind(c)) return 1;
  CK(launch_peer_meanfield(c));
  return 0;
}

int fmb200_peer_barrier(fmb200_ctx* c) {
  NEED_CTX(c);
  if (c->peer_world <= 1) return 0;
  if (bind(c)) return 1;
  CK(launch_peer_barrier(c));
  return 0;
}

int fmb200_stream(fmb200_ctx* c, void** cuda_stream) {
  NEED_CTX(c);
  if (cuda_stream) *cuda_stream = (void*)c->stream;
  return 0;
}

int fmb200_kernel_launches(fmb200_ctx* c, uint64_t* count) {
  NEED_CTX(c);
  if (count) *count = c->launches;
  return 0;
}

int fmb200_last_epoch_config(fmb200_ctx* c, int* lanes_per_row, int* slots, int* rows_per_tile,
                             int* grid, int* block, int* smem_bytes, int* damp) {
  NEED_CTX(c);
  if (lanes_per_row) *lanes_per_row = c->last_cfg.lanes_per_row;
  if (slots) *slots = c->last_cfg.slots;
  if (rows_per_tile) *rows_per_tile = c->last_cfg.rows_per_tile;
  if (grid) *grid = c->last_cfg.grid;
  if (block) *block = c->last_cfg.block;
  if (smem_bytes) *smem_bytes = c->last_cfg.smem;
  if (damp) *damp = c->last_cfg.damp;
  return 0;
}

int fmb200_last_epoch_dealt(fmb200_ctx* c, int* dealt) {
  NEED_CTX(c);
  if (dealt) *dealt = c->last_cfg.dealt;
  return 0;
}

int fmb200_download_data(fmb200_ctx* c, int slot, uint64_t* n_rows, uint64_t* nnz, uint64_t* row_ptr,
                         uint32_t* col, float* val, float* target) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  const DataSlot& d = c->slots[slot];
  if (n_rows) *n_rows = d.n_rows;
  if (nnz) *nnz = d.nnz;
  if (row_ptr) CK(cudaMemcpyAsync(row_ptr, d.row_ptr.get(), (d.n_rows + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
  if (col && d.nnz) CK(cudaMemcpyAsync(col, d.col.get(), d.nnz * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  if (val && d.nnz) CK(cudaMemcpyAsync(val, d.val.get(), d.nnz * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (target && d.n_rows) CK(cudaMemcpyAsync(target, d.target.get(), d.n_rows * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_ordered_index(fmb200_ctx* c, int slot, uint32_t* link, uint32_t* rowdep) {
  NEED_CTX(c);
  if (need_slot(c, slot)) return 1;
  if (bind(c)) return 1;
  DataSlot& d = c->slots[slot];
  if (d.nnz >= 0xffffffffull) return fail("the ORDERED index needs nnz < 2^32-1");
  CK(build_ordered_links(c, d));
  if (link && d.nnz)
    CK(cudaMemcpyAsync(link, d.link.get(), d.nnz * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  if (rowdep && d.n_rows)
    CK(cudaMemcpyAsync(rowdep, d.rowdep.get(), d.n_rows * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return 0;
}

int fmb200_set_tuning(fmb200_ctx* c, int ctas_per_sm, int rows_per_tile, int threads, int damp,
                      int variant) {
  NEED_CTX(c);
  if (threads && (threads % 32 != 0 || threads < 32 || threads > 1024))
    return fail("threads must be a multiple of 32 in [32,1024]");
  // the SGD epochs take the tile of 32 .. 512 rows nearest below it; HOGWILD SGDA takes it as its window, whose
  // fixed-point sums hold up to 2^20 rows
  if (rows_per_tile && (rows_per_tile < 1 || rows_per_tile > (1 << 20)))
    return fail("rows_per_tile must be in [1,2^20]");
  c->tune_ctas_per_sm = ctas_per_sm;
  c->tune_rows_per_tile = rows_per_tile;
  c->tune_threads = threads;
  c->tune_damp = damp;
  c->tune_variant = variant;
  return 0;
}

int fmb200_set_reproducible(fmb200_ctx* c, int on, int tile_rows, int window_tiles) {
  NEED_CTX(c);
  if (tile_rows < 0 || tile_rows > fmb::kWindowMaxTileRows) return fail("tile_rows must be in [1,1024] (0: 256)");
  if (window_tiles < 0 || window_tiles > fmb::kWindowMaxTiles)
    return fail("window_tiles must be in [1,65536] (0: 64)");
  c->win_on = on != 0;
  c->win_tile_rows = tile_rows ? tile_rows : (int)fmb::kWindowTileRows;
  c->win_tiles = window_tiles ? window_tiles : (int)fmb::kWindowTiles;
  return 0;
}

}  // extern "C"
