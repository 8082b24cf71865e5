// extern "C" surface declared in include/afl_b200.h, error plumbing, and the one-call host-buffer API.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "afl_common.cuh"

namespace afl {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d: %s", static_cast<int>(e), cudaGetErrorString(e), file, line, what);
  return AFL_ERR_CUDA;
}
void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

// ---- event-based kernel timing -----------------------------------------------------------------
struct ProfRec { std::string name; cudaEvent_t e0, e1; };
static std::atomic<int> g_prof_on{0};
static std::mutex g_prof_mu;
static std::vector<ProfRec*> g_prof_recs;

static bool dominant_kernel(const char* n) {
  return !strncmp(n, "gram_", 5) || !strcmp(n, "sqdist_simt") || !strcmp(n, "trimmed_mean") || !strcmp(n, "mean") || !strcmp(n, "alie");
}
ProfScope::ProfScope(const char* name, cudaStream_t stream) : name_(name), stream_(stream), rec_(nullptr) {
  const int mode = g_prof_on.load(std::memory_order_relaxed);
  if (!mode || (mode == 2 && !dominant_kernel(name))) return;
  ProfRec* r = new ProfRec{name, nullptr, nullptr};
  if (cudaEventCreate(&r->e0) != cudaSuccess || cudaEventCreate(&r->e1) != cudaSuccess) { delete r; return; }
  cudaEventRecord(r->e0, stream);
  rec_ = r;
}
ProfScope::~ProfScope() {
  if (!rec_) return;
  ProfRec* r = static_cast<ProfRec*>(rec_);
  cudaEventRecord(r->e1, stream_);
  std::lock_guard<std::mutex> lock(g_prof_mu);
  g_prof_recs.push_back(r);
}
static int profile_read(const char* kernel, double* total_ms, int* launches) {
  std::lock_guard<std::mutex> lock(g_prof_mu);
  double tot = 0.0; int cnt = 0;
  std::vector<ProfRec*> keep;
  for (ProfRec* r : g_prof_recs) {
    if (r->name != kernel) { keep.push_back(r); continue; }
    float ms = 0.f;
    cudaError_t e = cudaEventSynchronize(r->e1);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, r->e0, r->e1);
    cudaEventDestroy(r->e0); cudaEventDestroy(r->e1);
    delete r;
    if (e != cudaSuccess) return cuda_fail(e, "afl_profile_read", __FILE__, __LINE__);
    tot += ms; ++cnt;
  }
  g_prof_recs.swap(keep);
  if (total_ms) *total_ms = tot;
  if (launches) *launches = cnt;
  return AFL_OK;
}

// Per-device state: the C ABI promises "current device" semantics (afl_b200.h), so nothing below may
// remember the first device it saw.
int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
  return dev;
}
int sm_count() {
  static int cached[kMaxDevices] = {0};
  const int dev = current_device();
  if (!cached[dev]) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
      cached[dev] = sms;
    else
      return 132;   // H100 SXM; used only for workspace sizing when no device is visible
  }
  return cached[dev];
}

namespace gram {
size_t workspace_bytes(int n, int64_t d, int dtype, int flags);
size_t workspace_bytes(int n, int64_t d, int dtype, int flags, int batch);
int sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out, void* ws, size_t ws_bytes,
                   int flags, cudaStream_t stream);
int sqdist_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, double* d2_out,
                   void* ws, size_t ws_bytes, int flags, cudaStream_t stream, const ProblemParams* rows = nullptr);
int sqdist_to_dist(const double* d2, int n, float* dist, cudaStream_t stream, int batch = 1);
}
namespace select {
int max_clients();
size_t workspace_bytes(int n);
size_t workspace_bytes(int n, int batch);
int krum_select(const float* dist, int n, int users_count, int corrupted_count, int* idx_out, float* scores_out,
                void* ws, size_t ws_bytes, cudaStream_t stream);
int krum_from_sqdist(const double* d2, int n, int users_count, int corrupted_count, int* idx_out, void* ws,
                     size_t ws_bytes, cudaStream_t stream, int batch = 1, const ProblemParams* each = nullptr,
                     bool rows = false);
int bulyan_select(const float* dist, int n, int users_count, int f, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream, int batch = 1, const ProblemParams* each = nullptr);
int bulyan_rounds(const float* dist, int n, int f, int theta, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream, int batch, const ProblemParams* each, bool rows);
}
namespace tmean {
int trimmed_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                 int corrupted_count, float* out, cudaStream_t stream);
int trimmed_mean_batched(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                         int corrupted_count, float* out, int batch, int64_t g_batch, int ri_batch, int64_t out_batch,
                         cudaStream_t stream, const ProblemParams* each = nullptr);
int trimmed_mean_classes(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, float* out,
                         int batch, int64_t g_batch, int ri_batch, int64_t out_batch, cudaStream_t stream,
                         const ProblemParams* each, const int* perm, const int* counts);
int trimmed_mean_classes_dev(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, float* out,
                             int batch, int64_t g_batch, int ri_batch, int64_t out_batch, cudaStream_t stream,
                             const ProblemParams* each, const int* perm, const int* start);
}
namespace colstats {
int mean(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, cudaStream_t stream);
int mean_batched(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, int batch, int64_t g_batch,
                 int64_t out_batch, cudaStream_t stream, const ProblemParams* rows = nullptr);
int alie(const void* G, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
         float* crafted_out, float* bcast, int64_t bcast_ld, cudaStream_t stream);
int alie_batched(const void* G, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
                 float* crafted_out, float* bcast, int64_t bcast_ld, int batch, int64_t g_batch, int64_t out_batch,
                 int64_t bcast_batch, cudaStream_t stream, const ProblemParams* each = nullptr);
int alie_batched_dev(const void* G, int f_bound, int64_t d, int64_t ld, int dtype, float* mu_out, float* sigma_out,
                     float* crafted_out, void* bcast, int64_t bcast_ld, int batch, int64_t g_batch, int64_t out_batch,
                     int64_t bcast_batch, cudaStream_t stream, const ProblemParams* each);
int gather_row(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* idx_dev, float* out,
               cudaStream_t stream);
int momentum_step(float* w, float* v, const float* g, int64_t d, float momentum, float lr, cudaStream_t stream);
int momentum_step_batched(float* w, float* v, const float* g, int batch, int64_t d, float momentum, const float* lr,
                          cudaStream_t stream);
int alie_band(const float* mu, const float* sigma, double z, const float* x, float* out, int64_t d, cudaStream_t stream);
int64_t deviation_tiles(int64_t d, int dtype);
int attack_metrics(const void* G, int batch, int64_t g_batch, int n, int64_t d, int64_t ld, int dtype, int f,
                   const ProblemParams* each, const float* agg, const int* idx, const int* sel, int sel_ld,
                   float* dev_out, double* sums_out, float* honest_out, int* krum_hit, int* mal_count, int* sel_count,
                   void* partial, cudaStream_t stream, bool rows = false);
int attack_trace(const float* G, int batch, int64_t g_batch, int n, int64_t d, int64_t ld, const ProblemParams* each,
                 const float* agg, const int* idx, const int* sel, int sel_ld, const int* slot, int n_slots,
                 int64_t table_ld, float* agg_dev, float* mal_dev, int* idx_out, int* mal_count, int* sel_count,
                 void* partial, cudaStream_t stream, bool rows);
int backdoor_start(const void* G, int fmax, int64_t d, int64_t ld, int dtype, int batch, int64_t g_batch,
                   const ProblemParams* each, const float* w, int64_t w_batch, float* mu_out, float* sigma_out,
                   float* initial_out, cudaStream_t stream);
int backdoor_finish(int batch, int64_t d, const ProblemParams* each, const float* mu, const float* sigma,
                    const float* initial, const float* mal, int64_t mal_batch, float* crafted_out, float* bcast,
                    int64_t bcast_batch, int64_t bcast_ld, cudaStream_t stream);
}

__global__ void add_f64_kernel(double* __restrict__ acc, const double* __restrict__ x, size_t n, int first) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) acc[i] = first ? x[i] : acc[i] + x[i];
}

// ------------------------------------------------------------------------------------------------
// Host-buffer path: the matrix stays in host memory and is streamed through a bounded device staging area.
// Every host entry point (afl_defend_host, afl_sqdist_host, afl_bulyan_host, afl_alie_host) runs on the
// helpers below: one HostCall per call, one stage() for the budget and buffers, one slot ring.
//
//   * Column slabs of `slab_cols` columns go through a ring of kRingSlots device slots: the copy stream fills
//     slot s % slots while the compute stream runs the kernels of the slab before it.  `freed[slot]` is
//     recorded on the compute stream after the last kernel that reads the slot, and the copy stream waits on
//     it before overwriting the slot.
//   * Krum, Bulyan and afl_sqdist_host sum one d2 table per slab (sum_sqdist: sqdist_partial + add_f64_kernel,
//     in slab order); TrimmedMean and NoDefense finish each slab's columns as soon as its kernel has run.
//   * Bulyan keeps slabs 0 .. R-1 resident (as many as the budget holds) and streams the rest.  After
//     selection, stage 2 runs once over the resident columns with row_index = sel; for the other columns it
//     re-streams only the theta selected rows, packed in selection order, and runs the same trimmed mean with
//     row_index = NULL.  When the whole matrix fits, R covers every slab and nothing is streamed twice.
//   * ALIE packs the f separate user vectors of each slab into a slot (one copy per row) and runs the
//     column-wise alie kernel on it.
//   * Budget: free device memory plus what this context already holds, minus 1 GiB, capped by the
//     environment variable AFL_HOST_DEVICE_BYTES (read on every call).
//
// Results depend only on the input, n, d, ld and slab_cols: every kernel is column-wise or sums per-slab
// tables in slab order, so neither the budget, the ring depth nor the resident prefix changes a bit.  For the
// same reason the slab width is never narrowed to fit a small budget: the call fails instead.
// ------------------------------------------------------------------------------------------------
constexpr int kRingSlots = 3;
constexpr size_t kHeadroom = size_t(1) << 30;

struct HostCtx {
  std::mutex mu;
  void* stage = nullptr; size_t stage_bytes = 0;   // Bulyan's resident prefix, then the ring slots
  void* ws = nullptr; size_t ws_bytes = 0;          // kernel workspace
  void* small = nullptr; size_t small_bytes = 0;    // d2 tables, dist, indices, output vectors
  cudaStream_t copy = nullptr, comp = nullptr;
  cudaEvent_t ready = nullptr;                      // slab landed (recorded on copy, waited on at once by comp)
  cudaEvent_t freed[kRingSlots];                    // compute stream is done reading the slot
  bool init = false;
};
static HostCtx g_ctx[kMaxDevices];

static int ensure(void** p, size_t* have, size_t want) {
  if (*have >= want) return AFL_OK;
  if (*p) { cudaFree(*p); *p = nullptr; *have = 0; }
  AFL_CUDA(cudaMalloc(p, want));
  *have = want;
  return AFL_OK;
}

// Device bytes the host path may hold on this call.
static size_t host_budget(size_t free_b, size_t held) {
  size_t b = free_b + held > kHeadroom ? free_b + held - kHeadroom : 0;
  if (const char* e = getenv("AFL_HOST_DEVICE_BYTES")) {
    if (*e) {
      const unsigned long long cap = strtoull(e, nullptr, 10);
      if (cap < b) b = static_cast<size_t>(cap);
    }
  }
  return b;
}

// Columns per slab: slab_cols rounded up to a multiple of 32 (0 = about 96 MB of `rows` rows), never wider than
// the padded matrix.
static int64_t slab_width(int64_t slab_cols, int rows, int64_t d) {
  const int64_t ld_dev = (d + 31) / 32 * 32;
  if (slab_cols <= 0) slab_cols = (int64_t(96) << 20) / (static_cast<int64_t>(rows) * 4);
  slab_cols = (slab_cols + 31) / 32 * 32;
  if (slab_cols < 32) slab_cols = 32;
  return slab_cols > ld_dev ? ld_dev : slab_cols;
}

// One call's hold on the current device's context: the lock, the streams and events (created once), and on
// every return both streams drained, so that no copy still reads the caller's host buffers.
struct HostCall {
  HostCtx& c;
  std::lock_guard<std::mutex> lock;
  bool open = false;
  HostCall() : c(g_ctx[current_device()]), lock(c.mu) {}
  ~HostCall() {
    if (open) { cudaStreamSynchronize(c.copy); cudaStreamSynchronize(c.comp); }
  }
  int begin() {
    if (!c.init) {
      AFL_CUDA(cudaStreamCreateWithFlags(&c.copy, cudaStreamNonBlocking));
      AFL_CUDA(cudaStreamCreateWithFlags(&c.comp, cudaStreamNonBlocking));
      AFL_CUDA(cudaEventCreateWithFlags(&c.ready, cudaEventDisableTiming));
      for (auto& e : c.freed) AFL_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      c.init = true;
    }
    open = true;
    return AFL_OK;
  }
  // the copy stream has issued a slab: the compute stream waits for it before the slab's kernels
  cudaError_t landed() {
    cudaError_t e = cudaEventRecord(c.ready, c.copy);
    return e != cudaSuccess ? e : cudaStreamWaitEvent(c.comp, c.ready, 0);
  }
};

// The staging area of one call, carved out of HostCtx::stage: slabs 0 .. R-1 resident at pitch ld_res, then
// `slots` ring slots of slot_elems floats.
struct Staging {
  int nslab = 0, R = 0, slots = 0;
  int64_t ld_res = 0, d_res = 0;                     // resident pitch and columns
  float* res = nullptr;
  float* ring = nullptr;
  int64_t slot_elems = 0;
  int64_t issued = 0;                                // ring slabs issued so far

  // next ring slot: the copy stream waits until the compute stream has finished reading it
  cudaError_t next_slot(HostCtx& c, int* slot, float** m) {
    *slot = static_cast<int>(issued % slots);
    *m = ring + *slot * slot_elems;
    return issued++ >= slots ? cudaStreamWaitEvent(c.copy, c.freed[*slot], 0) : cudaSuccess;
  }
};

// Fits a call into the budget and sizes the cached buffers: ws_need + small_need bytes are always held, plus
// two or three ring slots of slot_rows x slab_cols floats.  With `resident` (Bulyan) the rest of the budget goes
// to leading slabs of the n-row matrix that stay on the device (all of them when the matrix fits); otherwise the
// ring gets a third slot when it fits.  `who` names the entry point in the error.
static int stage(const char* who, HostCtx& c, int n, int64_t d, int64_t slab_cols, int slot_rows, size_t ws_need,
                 size_t small_need, bool resident, Staging* st) {
  const int64_t ld_dev = (d + 31) / 32 * 32;          // padded pitch: TMA + 16-byte loads always apply
  const int nslab = static_cast<int>((d + slab_cols - 1) / slab_cols);
  const size_t slab_bytes = static_cast<size_t>(n) * slab_cols * sizeof(float);
  const size_t slot_bytes = align_up(static_cast<size_t>(slot_rows) * slab_cols * sizeof(float), 256);
  size_t free_b = 0, total_b = 0;
  AFL_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = host_budget(free_b, c.stage_bytes + c.ws_bytes + c.small_bytes);
  const size_t fixed = ws_need + small_need;
  const size_t full_res = align_up(static_cast<size_t>(n) * ld_dev * sizeof(float), 256);
  int R = 0, slots = 0;                               // resident slabs, ring slots
  if (resident && fixed + full_res <= budget) {
    R = nslab;
  } else {
    const int min_slots = nslab < 2 ? nslab : 2;
    if (fixed + min_slots * slot_bytes > budget) {
      set_error("%s: needs %zu bytes of device memory (%d staging slots of %zu bytes for %lld-column slabs, "
                "plus %zu bytes of tables and workspaces) but may use %zu (free memory less 1 GiB, capped by "
                "AFL_HOST_DEVICE_BYTES); use narrower slabs or a larger budget",
                who, fixed + min_slots * slot_bytes, min_slots, slot_bytes, static_cast<long long>(slab_cols), fixed,
                budget);
      return AFL_ERR_UNSUPPORTED;
    }
    slots = min_slots;
    if (resident) {                                   // spend the rest on resident slabs: they are not re-streamed
      const size_t spare = budget - fixed - slots * slot_bytes;
      const size_t fit = spare > 256 ? (spare - 256) / slab_bytes : 0;
      R = static_cast<int>(fit < static_cast<size_t>(nslab - 1) ? fit : static_cast<size_t>(nslab - 1));
    } else {
      const int most = nslab < kRingSlots ? nslab : kRingSlots;
      while (slots < most && fixed + (slots + 1) * slot_bytes <= budget) ++slots;
    }
  }
  const int64_t ld_res = R == nslab ? ld_dev : R * slab_cols;
  const size_t res_bytes = align_up(static_cast<size_t>(n) * ld_res * sizeof(float), 256);
  const size_t stage_need = res_bytes + slots * slot_bytes;

  // release cached buffers that are larger than this call needs when keeping them would exceed the budget
  void** bufs[3] = {&c.stage, &c.ws, &c.small};
  size_t* have[3] = {&c.stage_bytes, &c.ws_bytes, &c.small_bytes};
  const size_t want[3] = {stage_need, ws_need, small_need};
  size_t keep = 0;
  for (int i = 0; i < 3; ++i) keep += *have[i] > want[i] ? *have[i] : want[i];
  if (keep > budget)
    for (int i = 0; i < 3; ++i)
      if (*have[i] > want[i]) { AFL_CUDA(cudaFree(*bufs[i])); *bufs[i] = nullptr; *have[i] = 0; }
  for (int i = 0; i < 3; ++i) {
    const int rc = ensure(bufs[i], have[i], want[i]);
    if (rc) return rc;
  }
  st->nslab = nslab; st->R = R; st->slots = slots;
  st->ld_res = ld_res;
  st->d_res = R == nslab ? d : R * slab_cols;
  st->res = static_cast<float*>(c.stage);
  st->ring = reinterpret_cast<float*>(static_cast<uint8_t*>(c.stage) + res_bytes);
  st->slot_elems = static_cast<int64_t>(slot_bytes / sizeof(float));
  st->issued = 0;
  return AFL_OK;
}

// Pass 1: every column of the n x d host matrix G (pitch ld) once, slab by slab into the resident prefix or the
// ring.  kernel(m, mld, c0, w, s) enqueues slab s (columns c0 .. c0+w-1 at m, pitch mld) on the compute stream.
template <typename Kernel>
static int pass1(HostCall& call, Staging& st, const float* G, int n, int64_t d, int64_t ld, int64_t slab_cols,
                 Kernel kernel) {
  HostCtx& c = call.c;
  for (int s = 0; s < st.nslab; ++s) {
    const int64_t c0 = static_cast<int64_t>(s) * slab_cols;
    const int64_t w = (d - c0 < slab_cols) ? d - c0 : slab_cols;
    int slot = -1;
    float* m = st.res + c0;
    if (s >= st.R) AFL_CUDA(st.next_slot(c, &slot, &m));
    const int64_t mld = s < st.R ? st.ld_res : slab_cols;
    AFL_CUDA(cudaMemcpy2DAsync(m, mld * sizeof(float), G + c0, ld * sizeof(float), w * sizeof(float), n,
                               cudaMemcpyHostToDevice, c.copy));
    AFL_CUDA(call.landed());
    const int rc = kernel(m, mld, c0, w, s);
    if (rc) return rc;
    if (slot >= 0) AFL_CUDA(cudaEventRecord(c.freed[slot], c.comp));
  }
  return AFL_OK;
}

// Pass 1 into the summed n x n float64 d2 table: sqdist_partial per slab into d2_part, added into d2_acc in slab
// order.  Krum, Bulyan and afl_sqdist_host all build their table here.
static int sum_sqdist(HostCall& call, Staging& st, const float* G, int n, int64_t d, int64_t ld, int64_t slab_cols,
                      double* d2_acc, double* d2_part, void* gram_ws, size_t gram_ws_bytes) {
  const size_t nn = static_cast<size_t>(n) * n;
  cudaStream_t comp = call.c.comp;
  return pass1(call, st, G, n, d, ld, slab_cols, [&](const float* m, int64_t mld, int64_t, int64_t w, int s) -> int {
    const int rc = gram::sqdist_partial(m, n, w, mld, AFL_F32, d2_part, gram_ws, gram_ws_bytes, 0, comp);
    if (rc) return rc;
    add_f64_kernel<<<static_cast<unsigned>((nn + 255) / 256), 256, 0, comp>>>(d2_acc, d2_part, nn, s == 0);
    AFL_LAUNCH_CHECK("add_f64_kernel");
    return AFL_OK;
  });
}

static int sqdist_host(const float* G, int n, int64_t d, int64_t ld, double* d2_out, int64_t slab_cols) {
  if (!G || !d2_out || n < 1 || d < 1 || ld < d) { set_error("afl_sqdist_host: bad argument"); return AFL_ERR_BAD_ARG; }
  HostCall call;
  int rc = call.begin(); if (rc) return rc;
  slab_cols = slab_width(slab_cols, n, d);
  const size_t nn = static_cast<size_t>(n) * n;
  const size_t gram_ws_bytes = align_up(gram::workspace_bytes(n, slab_cols, AFL_F32, 0), 256);
  Staging st;
  rc = stage("afl_sqdist_host", call.c, n, d, slab_cols, n, gram_ws_bytes, align_up(nn * 8, 256), false, &st);
  if (rc) return rc;
  rc = sum_sqdist(call, st, G, n, d, ld, slab_cols, d2_out, static_cast<double*>(call.c.small), call.c.ws, gram_ws_bytes);
  if (rc) return rc;
  AFL_CUDA(cudaStreamSynchronize(call.c.comp));
  return AFL_OK;
}

static int bulyan_host(const char* who, const float* G, int n, int64_t d, int64_t ld, int users_count, int f,
                       float* out_host, int* sel_host, int64_t slab_cols) {
  if (!G || n < 1 || d < 1 || ld < d) { set_error("%s: bad argument", who); return AFL_ERR_BAD_ARG; }
  if (!out_host) { set_error("%s: out_host is required for Bulyan", who); return AFL_ERR_BAD_ARG; }
  if (users_count < 4 * f + 3) {                      // the reference's assert (defences.py:56)
    set_error("bulyan: users_count >= 4*corrupted_count + 3 violated (%d, %d)", users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if (n > select::max_clients()) {                    // before any copy or launch
    set_error("%s: Bulyan supports n <= %d clients (got %d)", who, select::max_clients(), n);
    return AFL_ERR_UNSUPPORTED;
  }
  HostCall call;
  int rc = call.begin(); if (rc) return rc;
  HostCtx& c = call.c;
  const int theta = users_count - 2 * f;
  slab_cols = slab_width(slab_cols, n, d);
  const size_t nn = static_cast<size_t>(n) * n;
  const int sel_len = n > theta ? n : theta;         // also the rows of a slot: the second pass packs theta rows
  const size_t gram_ws_bytes = align_up(gram::workspace_bytes(n, slab_cols, AFL_F32, 0), 256);
  const size_t small_need = align_up(nn * 8, 256) * 2 + align_up(nn * 4, 256) +
                            align_up(static_cast<size_t>(sel_len) * 4, 256) + align_up(static_cast<size_t>(d) * 4, 256) + 1024;
  Staging st;
  rc = stage(who, c, n, d, slab_cols, sel_len, gram_ws_bytes + select::workspace_bytes(n), small_need, true, &st);
  if (rc) return rc;
  uint8_t* sp = static_cast<uint8_t*>(c.small);
  double* d2_acc = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256);
  double* d2_part = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256);
  float* dist = reinterpret_cast<float*>(sp); sp += align_up(nn * 4, 256);
  int* sel = reinterpret_cast<int*>(sp); sp += align_up(static_cast<size_t>(sel_len) * 4, 256);
  float* out_dev = reinterpret_cast<float*>(sp);
  void* sel_ws = static_cast<uint8_t*>(c.ws) + gram_ws_bytes;
  const size_t sel_ws_bytes = c.ws_bytes - gram_ws_bytes;

  rc = sum_sqdist(call, st, G, n, d, ld, slab_cols, d2_acc, d2_part, c.ws, gram_ws_bytes); if (rc) return rc;
  rc = gram::sqdist_to_dist(d2_acc, n, dist, c.comp); if (rc) return rc;
  rc = select::bulyan_select(dist, n, users_count, f, sel, sel_ws, sel_ws_bytes, c.comp); if (rc) return rc;
  if (st.R > 0) {                                     // stage 2 over the resident columns
    rc = tmean::trimmed_mean(st.res, n, st.d_res, st.ld_res, AFL_F32, sel, theta, 2 * f, out_dev, c.comp);
    if (rc) return rc;
  }
  std::vector<int> hsel(static_cast<size_t>(theta));
  AFL_CUDA(cudaMemcpyAsync(hsel.data(), sel, static_cast<size_t>(theta) * sizeof(int), cudaMemcpyDeviceToHost, c.comp));
  AFL_CUDA(cudaStreamSynchronize(c.comp));
  if (sel_host) memcpy(sel_host, hsel.data(), static_cast<size_t>(theta) * sizeof(int));
  if (hsel[theta - 1] < 0) {                          // a failed round marks itself and every later round with -1
    set_error("bulyan: a selection round found no eligible user (NaN or >= 1e20 scores); the reference raises KeyError(-1)");
    return AFL_ERR_NO_WINNER;
  }
  // ---- pass 2: the theta selected rows of the streamed columns, packed in selection order.  The kernel is
  // column-wise, so the slab may be as wide as a slot holds.
  const int64_t w2 = st.slot_elems / theta / 32 * 32;
  for (int64_t c0 = st.d_res; c0 < d; c0 += w2) {
    const int64_t w = (d - c0 < w2) ? d - c0 : w2;
    int slot = -1;
    float* m = nullptr;
    AFL_CUDA(st.next_slot(c, &slot, &m));
    for (int i = 0; i < theta; ++i) {
      const int row = hsel[i] < 0 ? hsel[i] + n : hsel[i];
      AFL_CUDA(cudaMemcpyAsync(m + static_cast<int64_t>(i) * w2, G + static_cast<int64_t>(row) * ld + c0,
                               w * sizeof(float), cudaMemcpyHostToDevice, c.copy));
    }
    AFL_CUDA(call.landed());
    rc = tmean::trimmed_mean(m, theta, w, w2, AFL_F32, nullptr, theta, 2 * f, out_dev + c0, c.comp); if (rc) return rc;
    AFL_CUDA(cudaEventRecord(c.freed[slot], c.comp));
  }
  AFL_CUDA(cudaMemcpyAsync(out_host, out_dev, static_cast<size_t>(d) * sizeof(float), cudaMemcpyDeviceToHost, c.comp));
  AFL_CUDA(cudaStreamSynchronize(c.comp));
  return AFL_OK;
}

static int defend_host(const char* rule, const float* G, int n, int64_t d, int64_t ld, int users_count, int f,
                       float* out_host, int* idx_out, int64_t slab_cols) {
  enum { R_MEAN, R_KRUM, R_TM } r;
  if (!strcmp(rule, "NoDefense")) r = R_MEAN;
  else if (!strcmp(rule, "Krum")) r = R_KRUM;
  else if (!strcmp(rule, "TrimmedMean")) r = R_TM;
  else if (!strcmp(rule, "Bulyan")) {
    const int rc = bulyan_host("afl_defend_host", G, n, d, ld, users_count, f, out_host, nullptr, slab_cols);
    if (rc == AFL_OK && idx_out) *idx_out = -1;
    return rc;
  }
  else { set_error("afl_defend_host: unknown rule '%s'", rule); return AFL_ERR_BAD_ARG; }
  if (!G || n < 1 || d < 1 || ld < d) { set_error("afl_defend_host: bad argument"); return AFL_ERR_BAD_ARG; }
  if (r != R_KRUM && !out_host) { set_error("afl_defend_host: out_host is required for %s", rule); return AFL_ERR_BAD_ARG; }
  // the reference's assert (defences.py:24-25)
  if (r == R_KRUM && users_count < 2 * f + 1) {
    set_error("krum: users_count >= 2*corrupted_count + 1 violated (%d, %d)", users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if (r == R_KRUM && n > select::max_clients()) {   // before any copy or launch
    set_error("afl_defend_host: %s supports n <= %d clients (got %d)", rule, select::max_clients(), n);
    return AFL_ERR_UNSUPPORTED;
  }
  HostCall call;
  int rc = call.begin(); if (rc) return rc;
  HostCtx& c = call.c;
  const bool table = r == R_KRUM;
  slab_cols = slab_width(slab_cols, n, d);
  const size_t nn = static_cast<size_t>(n) * n;

  // ---- device footprint: workspaces and tables (fixed), then the ring
  const size_t gram_ws_bytes = table ? align_up(gram::workspace_bytes(n, slab_cols, AFL_F32, 0), 256) : 0;
  const size_t ws_need = table ? gram_ws_bytes + select::workspace_bytes(n) : 256;
  const size_t small_need = (table ? align_up(nn * 8, 256) * 2 + align_up(nn * 4, 256) : 0) +
                            align_up(static_cast<size_t>(n) * 4, 256) +
                            (r != R_KRUM ? align_up(static_cast<size_t>(d) * 4, 256) : 0) + 1024;
  Staging st;
  rc = stage("afl_defend_host", c, n, d, slab_cols, n, ws_need, small_need, false, &st);
  if (rc) return rc;

  uint8_t* sp = static_cast<uint8_t*>(c.small);
  if (r == R_KRUM) {
    double* d2_acc = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256);
    double* d2_part = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256) + align_up(nn * 4, 256);
    int* sel = reinterpret_cast<int*>(sp);
    rc = sum_sqdist(call, st, G, n, d, ld, slab_cols, d2_acc, d2_part, c.ws, gram_ws_bytes); if (rc) return rc;
    int host_idx = -1;
    rc = select::krum_from_sqdist(d2_acc, n, users_count, f, sel, static_cast<uint8_t*>(c.ws) + gram_ws_bytes,
                                  c.ws_bytes - gram_ws_bytes, c.comp);
    if (rc) return rc;
    AFL_CUDA(cudaMemcpyAsync(&host_idx, sel, sizeof(int), cudaMemcpyDeviceToHost, c.comp));
    AFL_CUDA(cudaStreamSynchronize(c.comp));
    if (idx_out) *idx_out = host_idx;
    if (out_host) {                                   // the reference returns the winning ROW (a view)
      const int row = host_idx < 0 ? host_idx + n : host_idx;
      memcpy(out_host, G + static_cast<int64_t>(row) * ld, static_cast<size_t>(d) * sizeof(float));
    }
    return AFL_OK;
  }
  float* out_dev = reinterpret_cast<float*>(sp + align_up(static_cast<size_t>(n) * 4, 256));
  rc = pass1(call, st, G, n, d, ld, slab_cols, [&](const float* m, int64_t mld, int64_t c0, int64_t w, int) -> int {
    if (r == R_TM) return tmean::trimmed_mean(m, n, w, mld, AFL_F32, nullptr, n, f, out_dev + c0, c.comp);
    return colstats::mean(m, n, w, mld, AFL_F32, out_dev + c0, c.comp);
  });
  if (rc) return rc;
  AFL_CUDA(cudaMemcpyAsync(out_host, out_dev, static_cast<size_t>(d) * sizeof(float), cudaMemcpyDeviceToHost, c.comp));
  AFL_CUDA(cudaStreamSynchronize(c.comp));
  if (idx_out) *idx_out = -1;
  return AFL_OK;
}

static int alie_host(const float* const* rows, int f, int64_t d, double z, float* mu_out, float* sigma_out,
                     float* crafted_out, int64_t slab_cols) {
  if (!rows || f < 1 || d < 1) { set_error("afl_alie_host: bad argument"); return AFL_ERR_BAD_ARG; }
  for (int i = 0; i < f; ++i)
    if (!rows[i]) { set_error("afl_alie_host: rows[%d] is NULL", i); return AFL_ERR_BAD_ARG; }
  HostCall call;
  int rc = call.begin(); if (rc) return rc;
  HostCtx& c = call.c;
  slab_cols = slab_width(slab_cols, f, d);
  // device copies of the outputs; crafted_out == mu_out shares one, the in-place aliasing afl_alie reproduces
  float* outs[3] = {mu_out, sigma_out, crafted_out != mu_out ? crafted_out : nullptr};
  const size_t vec_bytes = align_up(static_cast<size_t>(d) * 4, 256);
  size_t small_need = 1024;
  for (float* o : outs) small_need += o ? vec_bytes : 0;
  Staging st;
  rc = stage("afl_alie_host", c, f, d, slab_cols, f, 256, small_need, false, &st);
  if (rc) return rc;
  float* dev[3] = {nullptr, nullptr, nullptr};
  uint8_t* sp = static_cast<uint8_t*>(c.small);
  for (int k = 0; k < 3; ++k)
    if (outs[k]) { dev[k] = reinterpret_cast<float*>(sp); sp += vec_bytes; }
  float* crafted_dev = crafted_out == mu_out ? dev[0] : dev[2];

  // each slab: the f row segments packed into one slot at pitch slab_cols, then the column-wise alie kernel
  for (int64_t c0 = 0; c0 < d; c0 += slab_cols) {
    const int64_t w = (d - c0 < slab_cols) ? d - c0 : slab_cols;
    int slot = -1;
    float* m = nullptr;
    AFL_CUDA(st.next_slot(c, &slot, &m));
    for (int i = 0; i < f; ++i)
      AFL_CUDA(cudaMemcpyAsync(m + static_cast<int64_t>(i) * slab_cols, rows[i] + c0, w * sizeof(float),
                               cudaMemcpyHostToDevice, c.copy));
    AFL_CUDA(call.landed());
    rc = colstats::alie(m, f, w, slab_cols, AFL_F32, z, dev[0] ? dev[0] + c0 : nullptr, dev[1] ? dev[1] + c0 : nullptr,
                        crafted_dev ? crafted_dev + c0 : nullptr, nullptr, 0, c.comp);
    if (rc) return rc;
    AFL_CUDA(cudaEventRecord(c.freed[slot], c.comp));
  }
  for (int k = 0; k < 3; ++k)
    if (outs[k])
      AFL_CUDA(cudaMemcpyAsync(outs[k], dev[k], static_cast<size_t>(d) * sizeof(float), cudaMemcpyDeviceToHost, c.comp));
  AFL_CUDA(cudaStreamSynchronize(c.comp));
  return AFL_OK;
}

// ------------------------------------------------------------------------------------------------
// Batched device calls: `batch` same-shape problems of n <= 128 clients, problem b at G + b * batch_stride, each
// computed by the same kernels as one problem (the batch is a grid dimension), so every problem's result is the
// single call's.  Scratch per rule (the tables first, so that a caller can read them after the call):
//   Krum   [d2: batch x n x n float64][gram workspace][selection workspace]
//   Bulyan [d2: batch x n x n float64][dist: batch x n x n fp32][gram workspace][selection workspace]
// The per-problem calls (*_each) take corrupted_count (and ALIE's z) per problem.  Their host arrays become one
// ProblemParams row per problem (problem_row, the builder problem_table_kernel runs on the device) copied to the start
// of the workspace; the scalar call's layout follows it.  The scalar calls pass no table and run as they always have.
// The large calls (afl_defend_batched_large) take up to 1024 clients per problem: every Gram form is batched for any
// tile count, and the register-resident trimmed-mean kernels end at 1024 rows.
// ------------------------------------------------------------------------------------------------
constexpr int kBatchMaxClients = 128;            // one Gram tile
constexpr int kBatchLargeMaxClients = 1024;      // the largest register-resident trimmed-mean kernel (S = 32)
constexpr int kBatchMax = 65535;                 // grid y / z limit

// The rule of a batched call: the defences, then the attacks and the metrics, whose tables the same builders make.
enum BatchedRule { B_BAD, B_MEAN, B_KRUM, B_TM, B_BULYAN, T_ALIE, T_METRICS, T_BACKDOOR };
static BatchedRule batched_rule(const char* rule) {
  if (!rule) return B_BAD;
  if (!strcmp(rule, "NoDefense")) return B_MEAN;
  if (!strcmp(rule, "Krum")) return B_KRUM;
  if (!strcmp(rule, "TrimmedMean")) return B_TM;
  if (!strcmp(rule, "Bulyan")) return B_BULYAN;
  return B_BAD;
}

// The defence `rule` names; with `attacks` (afl_batched_table_dev) also "ALIE" and "AttackMetrics".
static int parse_rule(const char* who, const char* rule, bool attacks, BatchedRule* r) {
  *r = batched_rule(rule);
  if (attacks && rule && !strcmp(rule, "ALIE")) *r = T_ALIE;
  if (attacks && rule && !strcmp(rule, "AttackMetrics")) *r = T_METRICS;
  if (*r != B_BAD) return AFL_OK;
  set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)");
  return AFL_ERR_BAD_ARG;
}

// Problem b's table row, built by the host calls (upload_table) and by problem_table_kernel alike:
//   defences: m rows (rows_b, or n), users count uc and f; Bulyan's table for its second stage (`second`) holds the
//     trimmed mean of the theta_b selected rows with 2 f_b;
//   ALIE and the backdoor: f, (float)z and write, and the backdoor's (float)lr (ALIE's is 0, so the union's bits are);
//   the metrics: f and tm.n_rows = m, which a call without rows passes as 0 (its kernels read no row count).
__host__ __device__ inline ProblemParams problem_row(int rule, int m, int uc, int f, double z, double lr, bool second) {
  ProblemParams q{};
  q.f = f;
  if (rule == T_METRICS) {
    q.tm.n_rows = m;
  } else if (rule == T_ALIE || rule == T_BACKDOOR) {
    q.z = static_cast<float>(z);
    q.lr = static_cast<float>(lr);
    q.write = f > 0 && z != 0.0;                         // malicious.py:20-21: z == 0 computes the statistics only
  } else {
    q.take = select::krum_take(m, uc, f);
    q.theta = uc - 2 * f;
    q.tm = rule == B_BULYAN && second ? tmean::shape(q.theta, 2 * f) : tmean::shape(m, f);
  }
  return q;
}

// The reference's asserts (defences.py:24-25, 56) and Bulyan's users_count == rows for one problem of m rows, users
// count uc and corrupted count f: the host calls' check_problems and the device's problem_code.
__host__ __device__ inline int problem_assert(int rule, int m, int uc, int f) {
  if (rule == B_KRUM && uc < 2 * static_cast<int64_t>(f) + 1) return AFL_ERR_PRECONDITION;
  if (rule == B_BULYAN && uc < 4 * static_cast<int64_t>(f) + 3) return AFL_ERR_PRECONDITION;
  if (rule == B_BULYAN && uc != m) return AFL_ERR_UNSUPPORTED;
  return AFL_OK;
}

// Shape checks shared by the batched calls, before any CUDA call.  max_rows: one Gram tile for the defences and ALIE.
static int check_batch(const char* who, const void* G, int batch, int64_t batch_stride, int rows, int64_t d, int64_t ld,
                       int dtype, int max_rows = kBatchMaxClients) {
  if (!G || rows < 1 || d < 1 || ld < d) { set_error("%s: bad argument", who); return AFL_ERR_BAD_ARG; }
  if (batch < 1) { set_error("%s: batch must be >= 1 (got %d)", who, batch); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (rows > max_rows) {
    set_error("%s: batched problems support n <= %d clients (got %d)", who, max_rows, rows);
    return AFL_ERR_UNSUPPORTED;
  }
  if (batch > 1 && batch_stride < static_cast<int64_t>(rows - 1) * ld + d) {
    set_error("%s: batch_stride %lld is negative or makes problems overlap (a problem spans %lld elements)", who,
              static_cast<long long>(batch_stride), static_cast<long long>(static_cast<int64_t>(rows - 1) * ld + d));
    return AFL_ERR_BAD_ARG;
  }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("%s: dtype", who); return AFL_ERR_UNSUPPORTED; }
  return AFL_OK;
}

static int check_workspace(const char* who, const void* ws, size_t ws_bytes, size_t need) {
  if (ws && ws_bytes >= need && reinterpret_cast<uintptr_t>(ws) % 256 == 0) return AFL_OK;
  set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, need);
  return AFL_ERR_WORKSPACE;
}

// Per-problem counts: non-NULL, each in [0, f_cap]; their range in *fmin, *fmax.
static int check_counts(const char* who, const int* fs, int batch, int f_cap, int* fmin, int* fmax) {
  if (!fs) { set_error("%s: the per-problem corrupted counts are NULL", who); return AFL_ERR_BAD_ARG; }
  *fmin = fs[0]; *fmax = fs[0];
  for (int b = 0; b < batch; ++b) {
    if (fs[b] < 0 || fs[b] > f_cap) {
      set_error("%s: corrupted count %d of problem %d is outside [0, %d]", who, fs[b], b, f_cap);
      return AFL_ERR_BAD_ARG;
    }
    *fmin = fs[b] < *fmin ? fs[b] : *fmin;
    *fmax = fs[b] > *fmax ? fs[b] : *fmax;
  }
  return AFL_OK;
}

// The per-problem checks of the host-array defences and metrics, each phase up to its first failing problem: the
// arrays are non-NULL (with `ragged`, rows and ucs too), every f_b is in [0, f_cap], every rows_b in [1, n], then the
// caller's outputs(), then problem_assert.  fs == NULL: the scalar call's f in every problem; rows == NULL: n rows;
// ucs == NULL: users_count.  Without rows, Bulyan's users_count == n is one condition of the call, checked after every
// problem's asserts.  The smallest f_b goes to *fmin, Bulyan's largest theta_b to *theta_max.
template <typename Outputs>
static int check_problems(const char* who, BatchedRule rule, int batch, int n, int f_cap, bool ragged, const int* rows,
                          const int* ucs, int users_count, const int* fs, int f, Outputs outputs, int* fmin,
                          int* theta_max) {
  if (ragged && (!rows || !ucs)) {
    set_error("%s: the per-problem row counts or users counts are NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  int fmax = f, rc = AFL_OK;
  *fmin = f;
  if ((fs || ragged) && (rc = check_counts(who, fs, batch, f_cap, fmin, &fmax))) return rc;
  for (int b = 0; rows && b < batch; ++b)
    if (rows[b] < 1 || rows[b] > n) {
      set_error("%s: row count %d of problem %d is outside [1, %d]", who, rows[b], b, n);
      return AFL_ERR_BAD_ARG;
    }
  if ((rc = outputs())) return rc;
  *theta_max = 0;
  for (int b = 0; b < batch; ++b) {
    const int m = rows ? rows[b] : n, uc = ucs ? ucs[b] : users_count, fb = fs ? fs[b] : f;
    const int code = problem_assert(rule, m, uc, fb);
    if (code == AFL_ERR_PRECONDITION) {
      const char* what = rule == B_KRUM ? "krum: users_count >= 2*corrupted_count + 1"
                                        : "bulyan: users_count >= 4*corrupted_count + 3";
      if (fs) set_error("%s violated (%d, %d) in problem %d", what, uc, fb, b);
      else set_error("%s violated (%d, %d)", what, uc, fb);
      return code;
    }
    if (code == AFL_ERR_UNSUPPORTED && rows) {
      set_error("%s: Bulyan's users_count (%d) must equal the number of rows (%d) in problem %d", who, uc, m, b);
      return code;
    }
    if (rule == B_BULYAN && uc - 2 * fb > *theta_max) *theta_max = uc - 2 * fb;
  }
  if (rule == B_BULYAN && !rows && users_count != n) {
    set_error("%s: Bulyan's users_count (%d) must equal the number of rows (%d)", who, users_count, n);
    return AFL_ERR_UNSUPPORTED;
  }
  return AFL_OK;
}

// The outputs a defence writes: out (all but Krum), idx_out (Krum), sel_out (Bulyan).  The scalar call's negative
// corrupted_count f is refused with the same message.
static int check_outputs(const char* who, const char* rule, BatchedRule r, const float* out, const int* idx_out,
                         const int* sel_out, int f = 0) {
  if ((r != B_KRUM && !out) || (r == B_KRUM && !idx_out) || (r == B_BULYAN && !sel_out) || f < 0) {
    set_error("%s: %s needs %s", who, rule, r == B_KRUM ? "idx_out" : r == B_BULYAN ? "out and sel_out" : "out");
    return AFL_ERR_BAD_ARG;
  }
  return AFL_OK;
}

// Rows 0 .. rows_max - 1 of every problem written at bcast_ld / bcast_batch_stride must not overlap.
static int check_bcast(const char* who, const void* bcast_rows, int rows_max, int64_t d, int batch,
                       int64_t bcast_batch_stride, int64_t bcast_ld) {
  if (bcast_rows && rows_max > 0 &&
      (bcast_ld < d || (batch > 1 && bcast_batch_stride < static_cast<int64_t>(rows_max - 1) * bcast_ld + d))) {
    set_error("%s: bcast_ld / bcast_batch_stride make the written rows overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  return AFL_OK;
}

static size_t table_bytes(int batch) { return align_up(static_cast<size_t>(batch) * sizeof(ProblemParams), 256); }
// The table of a batch with more than kBatchMaxClients rows per slot: ProblemParams[batch], then int perm[batch], the
// problems grouped by trimmed-mean slot class (tmean::trimmed_mean_classes).
static size_t class_table_bytes(int batch, int n) {
  if (n <= kBatchMaxClients) return table_bytes(batch);
  return align_up(static_cast<size_t>(batch) * (sizeof(ProblemParams) + sizeof(int)), 256);
}

// The rule's scratch after the table, in this order: d², Bulyan's dist, the Gram workspace, the selection workspace
// (bytes == 0: the rule needs none).  With `at`, the parts' addresses in a workspace whose scratch starts there.
struct RuleScratch {
  size_t bytes = 0, gram_bytes = 0, sel_bytes = 0;
  double* d2 = nullptr;
  float* dist = nullptr;
  void* gram = nullptr;
  void* sel = nullptr;
};
static RuleScratch rule_scratch(BatchedRule r, int batch, int n, int64_t d, int dtype, void* at = nullptr) {
  RuleScratch s;
  if (r != B_KRUM && r != B_BULYAN) return s;
  const size_t nn = static_cast<size_t>(batch) * n * n;
  const size_t tabs = align_up(nn * 8, 256) + (r == B_BULYAN ? align_up(nn * 4, 256) : 0);
  s.gram_bytes = align_up(gram::workspace_bytes(n, d, dtype, 0, batch), 256);
  s.sel_bytes = select::workspace_bytes(n, batch);
  s.bytes = tabs + s.gram_bytes + s.sel_bytes;
  if (uint8_t* p = static_cast<uint8_t*>(at)) {
    s.d2 = reinterpret_cast<double*>(p);
    s.dist = reinterpret_cast<float*>(p + align_up(nn * 8, 256));
    s.gram = p + tabs;
    s.sel = p + tabs + s.gram_bytes;
  }
  return s;
}

// The table of rows row(b), b < batch, copied to the workspace start (pageable source: the copy has taken the values
// when cudaMemcpyAsync returns).  With counts, the same copy appends int perm[batch]: the problems grouped by the
// trimmed-mean slot class of their tm.n_rows, in problem order within a class, whose sizes go to counts[kSlotClasses]
// (host).
template <typename Row>
static int upload_table(int batch, void* ws, cudaStream_t stream, Row row, int* counts = nullptr) {
  const size_t nb = static_cast<size_t>(batch);
  std::vector<ProblemParams> host(nb);
  for (int b = 0; b < batch; ++b) host[b] = row(b);
  if (!counts) {
    AFL_CUDA(cudaMemcpyAsync(ws, host.data(), nb * sizeof(ProblemParams), cudaMemcpyHostToDevice, stream));
    return AFL_OK;
  }
  std::vector<int> cls(nb), order(nb);
  for (int c = 0; c < kSlotClasses; ++c) counts[c] = 0;
  for (int b = 0; b < batch; ++b) {
    cls[b] = tmean::slot_class(host[b].tm.n_rows);
    ++counts[cls[b]];
  }
  int start[kSlotClasses];
  for (int c = 0, s = 0; c < kSlotClasses; s += counts[c], ++c) start[c] = s;
  for (int b = 0; b < batch; ++b) order[start[cls[b]]++] = b;          // problems in order within a class
  std::vector<uint8_t> bytes(nb * (sizeof(ProblemParams) + sizeof(int)));
  memcpy(bytes.data(), host.data(), nb * sizeof(ProblemParams));
  memcpy(bytes.data() + nb * sizeof(ProblemParams), order.data(), nb * sizeof(int));
  AFL_CUDA(cudaMemcpyAsync(ws, bytes.data(), bytes.size(), cudaMemcpyHostToDevice, stream));
  return AFL_OK;
}

// The host-array defences: afl_defend_batched (fs == NULL: the scalar f), _each (rows == NULL: n rows and users_count in
// every problem), _rows and _large (`ragged`: rows_b and users_count_b per problem; the large call passes rows = n when
// it gets none).  Every check runs before any CUDA call.  Problem b's row is problem_row on (rows_b, users_count_b,
// f_b); NoDefense without rows takes no table, as it ignores f.  Each kernel of a ragged batch reads the problem's row
// count from the table: tm.n_rows (the Gram centre, Krum, TrimmedMean, NoDefense), theta + 2f (Bulyan's selection,
// whose users_count is its row count).  Bulyan's second stage needs tm = shape(theta_b, 2 f_b): without rows the one
// table holds it; with rows a second upload replaces the first after the selection kernels, in stream order.  Slots of
// more than kBatchMaxClients rows append the class permutation to the table (class_table_bytes), and the trimmed mean
// runs one launch per class (tmean::trimmed_mean_classes).
static int defend_batched(const char* who, int max_clients, bool ragged, const char* rule, const void* G, int batch,
                          int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, const int* rows,
                          const int* ucs, int users_count, const int* fs, int f, float* out, int* idx_out,
                          int* sel_out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  BatchedRule r;
  int rc = parse_rule(who, rule, false, &r);
  if (rc || (rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, max_clients))) return rc;
  int fmin = 0, theta_max = 0;
  rc = check_problems(who, r, batch, n, INT32_MAX / 4, ragged, rows, ucs, users_count, fs, f,
                      [&] { return check_outputs(who, rule, r, out, idx_out, sel_out, f); }, &fmin, &theta_max);
  if (rc) return rc;
  const bool table = fs && (rows || r != B_MEAN), classes = n > kBatchMaxClients;
  const size_t tab_bytes = table ? class_table_bytes(batch, n) : 0;
  const RuleScratch s = rule_scratch(r, batch, n, d, dtype, static_cast<uint8_t*>(ws) + tab_bytes);
  if (tab_bytes + s.bytes > 0 && (rc = check_workspace(who, ws, ws_bytes, tab_bytes + s.bytes))) return rc;
  const ProblemParams* each = table ? static_cast<const ProblemParams*>(ws) : nullptr;
  const int* perm = classes ? reinterpret_cast<const int*>(each + batch) : nullptr;
  int counts[kSlotClasses];
  auto upload = [&](bool second) {
    return upload_table(batch, ws, stream, [&](int b) {
      return problem_row(r, rows ? rows[b] : n, ucs ? ucs[b] : users_count, fs[b], 0.0, 0.0, second);
    }, classes ? counts : nullptr);
  };
  if (table && (rc = upload(!rows))) return rc;
  if (r == B_MEAN) return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream, each);
  if (r == B_TM && classes)
    return tmean::trimmed_mean_classes(G, n, d, ld, dtype, nullptr, out, batch, batch_stride, 0, d, stream, each, perm,
                                       counts);
  if (r == B_TM)
    return tmean::trimmed_mean_batched(G, n, d, ld, dtype, nullptr, n, fmin, out, batch, batch_stride, 0, d, stream, each);
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, s.d2, s.gram, s.gram_bytes, 0, stream,
                            rows ? each : nullptr);
  if (rc) return rc;
  if (r == B_KRUM)                                       // a ragged table's take stands for users_count and f
    return select::krum_from_sqdist(s.d2, n, rows ? 0 : users_count, rows ? 0 : fmin, idx_out, s.sel, s.sel_bytes,
                                    stream, batch, each, rows != nullptr);
  if ((rc = gram::sqdist_to_dist(s.d2, n, s.dist, stream, batch))) return rc;
  rc = select::bulyan_rounds(s.dist, n, fmin, theta_max, sel_out, s.sel, s.sel_bytes, stream, batch, each,
                             rows != nullptr);
  if (rc || (rows && (rc = upload(true)))) return rc;
  if (classes)
    return tmean::trimmed_mean_classes(G, n, d, ld, dtype, sel_out, out, batch, batch_stride, theta_max, d, stream, each,
                                       perm, counts);
  return tmean::trimmed_mean_batched(G, n, d, ld, dtype, sel_out, theta_max, 2 * fmin, out, batch, batch_stride, theta_max,
                                     d, stream, each);
}

// fs == NULL: rows 0..f-1 and z in every problem of f-row problems (afl_alie_batched).  Otherwise problem b has n rows of
// which fs[b] are malicious, and its own z (afl_alie_batched_each); the workspace holds the table.
// max_rows: kBatchMaxClients, or no limit for afl_alie_batched_large (a column pass, as the backdoor's).
static int alie_batched(const char* who, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                        int dtype, int f, double z, const int* fs, const double* zs, float* mu_out, float* sigma_out,
                        float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* ws,
                        size_t ws_bytes, cudaStream_t stream, int max_rows = kBatchMaxClients) {
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, max_rows);
  if (rc) return rc;
  int fmin = f, fmax = f;
  if (fs) {
    if (!zs) { set_error("%s: the per-problem attack strengths are NULL", who); return AFL_ERR_BAD_ARG; }
    if ((rc = check_counts(who, fs, batch, n, &fmin, &fmax))) return rc;
  }
  if ((rc = check_bcast(who, bcast_rows, fmax, d, batch, bcast_batch_stride, bcast_ld))) return rc;
  if (fs) {
    if ((rc = check_workspace(who, ws, ws_bytes, table_bytes(batch)))) return rc;
    rc = upload_table(batch, ws, stream, [&](int b) { return problem_row(T_ALIE, 0, 0, fs[b], zs[b], 0.0, false); });
    if (rc) return rc;
  }
  return colstats::alie_batched(G, fmax, d, ld, dtype, z, mu_out, sigma_out, crafted_out, bcast_rows, bcast_ld, batch,
                                batch_stride, d, bcast_batch_stride, stream,
                                fs ? static_cast<const ProblemParams*>(ws) : nullptr);
}

// Attack-success metrics of a batch (afl_attack_metrics_batched; fs != NULL: afl_attack_metrics_batched_each).
// Workspace: [ProblemParams table][partial sums: double2[batch][tiles]]; the scalar call leaves the table unused.
static size_t metrics_partial_bytes(int batch, int64_t d, int dtype) {
  return align_up(static_cast<size_t>(batch) * colstats::deviation_tiles(d, dtype) * sizeof(double2), 256);
}

// The selection inputs of the metrics: the counts need sel, whose rows are sel_ld >= 1 apart.
static int check_sel(const char* who, const int* sel, int sel_ld, const int* mal_count, const int* sel_count) {
  if ((mal_count || sel_count) && !sel) { set_error("%s: mal_count and sel_count need sel", who); return AFL_ERR_BAD_ARG; }
  if (sel && sel_ld < 1) { set_error("%s: sel_ld must be >= 1 (got %d)", who, sel_ld); return AFL_ERR_BAD_ARG; }
  return AFL_OK;
}

// The metrics' pointer rules: the aggregate as agg or as idx, not both, and each output with the input it needs.
static int check_metrics_inputs(const char* who, const float* agg, const int* idx, const int* sel, int sel_ld,
                                const float* dev_out, const double* sums_out, const int* krum_hit, const int* mal_count,
                                const int* sel_count) {
  if (agg && idx) { set_error("%s: give the aggregate as agg or as idx, not both", who); return AFL_ERR_BAD_ARG; }
  if ((dev_out || sums_out) && !agg && !idx) {
    set_error("%s: dev_out and sums_out need an aggregate (agg or idx)", who);
    return AFL_ERR_BAD_ARG;
  }
  if (krum_hit && !idx) { set_error("%s: krum_hit needs idx", who); return AFL_ERR_BAD_ARG; }
  return check_sel(who, sel, sel_ld, mal_count, sel_count);
}

// rows != NULL (afl_attack_metrics_batched_rows, fs required): problem b has rows[b] rows, in [1, n].
static int attack_metrics(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, int f,
                          const int* fs, const float* agg, const int* idx, const int* sel, int sel_ld, float* dev_out,
                          double* sums_out, float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* ws,
                          size_t ws_bytes, cudaStream_t stream, const int* rows = nullptr) {
  const char* who = rows ? "afl_attack_metrics_batched_rows" : fs ? "afl_attack_metrics_batched_each" : "afl_attack_metrics_batched";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc) return rc;
  int fmin = 0, theta_max = 0;
  rc = check_problems(who, T_METRICS, batch, n, INT32_MAX, false, rows, nullptr, 0, fs, f, [&]() -> int {
    if (f < 0) { set_error("%s: corrupted_count %d is negative", who, f); return AFL_ERR_BAD_ARG; }
    return check_metrics_inputs(who, agg, idx, sel, sel_ld, dev_out, sums_out, krum_hit, mal_count, sel_count);
  }, &fmin, &theta_max);
  if (rc) return rc;
  const bool pass = dev_out || sums_out || honest_out;          // the column pass and its partial sums
  const size_t need = table_bytes(batch) + metrics_partial_bytes(batch, d, dtype);
  if ((fs || pass) && (rc = check_workspace(who, ws, ws_bytes, need))) return rc;
  if (fs) {
    rc = upload_table(batch, ws, stream, [&](int b) {
      return problem_row(T_METRICS, rows ? rows[b] : 0, 0, fs[b], 0.0, 0.0, false);
    });
    if (rc) return rc;
  }
  return colstats::attack_metrics(G, batch, batch_stride, n, d, ld, dtype, f,
                                  fs ? static_cast<const ProblemParams*>(ws) : nullptr, agg, idx, sel, sel_ld, dev_out,
                                  sums_out, honest_out, krum_hit, mal_count, sel_count,
                                  static_cast<uint8_t*>(ws) + table_bytes(batch), stream, rows != nullptr);
}

// The backdoor crafting's own arguments.  Start: w and every output, and w_batch_stride 0 (one shared w) or >= d.
static int check_backdoor_start(const char* who, int64_t d, const float* w, int64_t w_batch_stride, const float* mu_out,
                                const float* sigma_out, const float* initial_out) {
  if (!w || !mu_out || !sigma_out || !initial_out) { set_error("%s: w and every output are required", who); return AFL_ERR_BAD_ARG; }
  if (w_batch_stride < 0 || (w_batch_stride > 0 && w_batch_stride < d)) {
    set_error("%s: w_batch_stride %lld must be 0 (one shared w) or >= d", who, static_cast<long long>(w_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  return AFL_OK;
}

// Finish: 1 <= batch <= kBatchMax, and the problems' trained vectors mal do not overlap.
static int check_backdoor_finish(const char* who, int batch, int64_t d, int64_t mal_batch_stride) {
  if (batch < 1) { set_error("%s: batch must be >= 1 (got %d)", who, batch); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (batch > 1 && mal_batch_stride < d) {
    set_error("%s: mal_batch_stride %lld makes problems overlap", who, static_cast<long long>(mal_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  return AFL_OK;
}

// The backdoor's per-problem values (afl_backdoor_start_batched / _finish_batched): non-NULL, counts in [0, f_cap].
static int backdoor_values(const char* who, int batch, const int* fs, int f_cap, const double* zs, const double* lrs,
                           int* fmax) {
  if (!zs || !lrs) { set_error("%s: the per-problem attack strengths or learning rates are NULL", who); return AFL_ERR_BAD_ARG; }
  int fmin = 0;
  return check_counts(who, fs, batch, f_cap, &fmin, fmax);
}

// Their table (f, (float)z, (float)lr, write) at the start of the workspace: the calls' first CUDA call.
static int backdoor_table(const char* who, int batch, const int* fs, const double* zs, const double* lrs, void* ws,
                          size_t ws_bytes, cudaStream_t stream) {
  const int rc = check_workspace(who, ws, ws_bytes, table_bytes(batch));
  if (rc) return rc;
  return upload_table(batch, ws, stream, [&](int b) { return problem_row(T_BACKDOOR, 0, 0, fs[b], zs[b], lrs[b], false); });
}

static int backdoor_start(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                          const int* fs, const double* zs, const double* lrs, const float* w, int64_t w_batch_stride,
                          float* mu_out, float* sigma_out, float* initial_out, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
  const char* who = "afl_backdoor_start_batched";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc || (rc = check_backdoor_start(who, d, w, w_batch_stride, mu_out, sigma_out, initial_out))) return rc;
  int fmax = 0;
  if ((rc = backdoor_values(who, batch, fs, n, zs, lrs, &fmax))) return rc;
  if ((rc = backdoor_table(who, batch, fs, zs, lrs, ws, ws_bytes, stream))) return rc;
  return colstats::backdoor_start(G, fmax, d, ld, dtype, batch, batch_stride, static_cast<const ProblemParams*>(ws), w,
                                  w_batch_stride, mu_out, sigma_out, initial_out, stream);
}

static int backdoor_finish(int batch, int64_t d, const int* fs, const double* zs, const double* lrs, const float* mu,
                           const float* sigma, const float* initial, const float* mal, int64_t mal_batch_stride,
                           float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* ws,
                           size_t ws_bytes, cudaStream_t stream) {
  const char* who = "afl_backdoor_finish_batched";
  if (!mu || !sigma || !initial || !mal || !crafted_out || d < 1) { set_error("%s: bad argument", who); return AFL_ERR_BAD_ARG; }
  int rc = check_backdoor_finish(who, batch, d, mal_batch_stride);
  if (rc) return rc;
  int fmax = 0;
  if ((rc = backdoor_values(who, batch, fs, INT32_MAX, zs, lrs, &fmax))) return rc;
  if ((rc = check_bcast(who, bcast_rows, fmax, d, batch, bcast_batch_stride, bcast_ld))) return rc;
  if ((rc = backdoor_table(who, batch, fs, zs, lrs, ws, ws_bytes, stream))) return rc;
  return colstats::backdoor_finish(batch, d, static_cast<const ProblemParams*>(ws), mu, sigma, initial, mal,
                                   mal_batch_stride, crafted_out, bcast_rows, bcast_batch_stride, bcast_ld, stream);
}

// ------------------------------------------------------------------------------------------------
// Device-parameter calls (afl_*_dev): the per-problem arrays are device memory, so a call never reads them on the host.
// problem_table_kernel runs the host calls' per-problem checks in the same order (problem_code, whose asserts are
// problem_assert) and builds their rows with problem_row, one thread per problem.  A problem that fails a check gets
// its first code in the caller's sticky status[b] and the safe row of rows_b = n, users_count_b = n, f_b = 0, which
// keeps every kernel inside its slot; its outputs are then not the reference's, and only status says so.  After the
// host checks of shapes, pointers and the workspace, a call makes no host copy, synchronisation or allocation, so it
// can be captured into a CUDA graph.
// ------------------------------------------------------------------------------------------------
struct TableArgs {
  int rule;                   // a BatchedRule
  int batch, n;
  const int* rows;            // NULL: n rows in every problem
  const int* ucs;             // NULL: users_count without rows, rows with them
  int users_count;
  const int* fs;
  const double* zs;           // ALIE and the backdoor only
  const double* lrs;          // the backdoor only
  ProblemParams* table;
  int* status;
  const int* sel;             // Bulyan's second stage: rows of sel_ld entries, sel[b][theta_b - 1] < 0 = failed round
  int sel_ld;
};

static TableArgs table_args(BatchedRule rule, int batch, int n, const int* fs, void* ws, int* status) {
  TableArgs a{};
  a.rule = rule; a.batch = batch; a.n = n; a.fs = fs; a.table = static_cast<ProblemParams*>(ws); a.status = status;
  return a;
}

// The first code of the host calls' checks for one problem: afl_defend_batched_rows / _each (rows = n),
// afl_alie_batched_each, afl_attack_metrics_batched_rows / _each, and the backdoor's (ALIE's count range).
__device__ int problem_code(int rule, int n, bool ragged, int m, int uc, int f) {
  if (rule == T_ALIE || rule == T_BACKDOOR) return f < 0 || f > n ? AFL_ERR_BAD_ARG : AFL_OK;
  if (f < 0 || (rule != T_METRICS && f > INT32_MAX / 4)) return AFL_ERR_BAD_ARG;
  if (ragged && (m < 1 || m > n)) return AFL_ERR_BAD_ARG;
  return problem_assert(rule, m, uc, f);
}

__global__ void __launch_bounds__(128) problem_table_kernel(const TableArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.batch) return;
  int f = a.fs[b];
  int m = a.rows ? a.rows[b] : a.n;
  int uc = a.ucs ? a.ucs[b] : a.rows ? m : a.users_count;
  const int code = problem_code(a.rule, a.n, a.rows != nullptr, m, uc, f);
  if (code != AFL_OK) { m = a.n; uc = a.n; f = 0; }
  // Bulyan's second stage: the table after the selection, or the whole-slot call's only table
  const ProblemParams q = problem_row(a.rule, (a.rows || a.rule != T_METRICS) ? m : 0, uc, f, a.zs ? a.zs[b] : 0.0,
                                      a.lrs ? a.lrs[b] : 0.0, a.sel || !a.rows);
  a.table[b] = q;
  int st = code;
  if (st == AFL_OK && a.sel && a.sel[static_cast<int64_t>(b) * a.sel_ld + q.theta - 1] < 0) st = AFL_ERR_NO_WINNER;
  if (st != AFL_OK && a.status[b] == AFL_OK) a.status[b] = st;
}

static int launch_table(const TableArgs& a, cudaStream_t stream) {
  problem_table_kernel<<<static_cast<unsigned>((a.batch + 127) / 128), 128, 0, stream>>>(a);
  AFL_LAUNCH_CHECK("problem_table_kernel");
  return AFL_OK;
}

// The problems of a table grouped by the trimmed-mean slot class of their tm.n_rows, on the device: perm[batch] lists
// them class by class and in problem order within a class (upload_table's order), and start[kSlotClasses + 1]
// holds the offset of each class in perm.  One CTA walks the problems in chunks of its size: a first pass counts the
// classes (__syncthreads_count), a second places each problem at its class's running offset plus its rank in the
// chunk (warp ballots, then the counts of the warps before it).  No atomics and no waits between CTAs, so the order is
// stable and deterministic.  A flagged problem carries the safe row and falls into the class of its row count.
constexpr int kPermThreads = 1024;
constexpr size_t kClassStartBytes = 256;         // start[kSlotClasses + 1] at the end of a large _dev workspace

__device__ __forceinline__ int class_of(const ProblemParams* table, int b) {
  const int c = tmean::slot_class(table[b].tm.n_rows);
  return c < 0 ? 0 : c >= kSlotClasses ? kSlotClasses - 1 : c;
}

__global__ void __launch_bounds__(kPermThreads) class_perm_kernel(const ProblemParams* table, int batch, int* perm,
                                                                  int* start) {
  __shared__ int base[kSlotClasses];
  __shared__ int wcount[kPermThreads / 32][kSlotClasses];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int count = 0;                                        // thread c < kSlotClasses: the size of class c
  for (int b0 = 0; b0 < batch; b0 += kPermThreads) {
    const int c = b0 + tid < batch ? class_of(table, b0 + tid) : -1;
#pragma unroll
    for (int k = 0; k < kSlotClasses; ++k) {
      const int n = __syncthreads_count(c == k);
      if (tid == k) count += n;
    }
  }
  if (tid < kSlotClasses) base[tid] = count;
  __syncthreads();
  if (tid == 0) {
    int s = 0;
    for (int k = 0; k < kSlotClasses; ++k) {
      const int n = base[k];
      base[k] = s; start[k] = s;
      s += n;
    }
    start[kSlotClasses] = s;
  }
  __syncthreads();
  for (int b0 = 0; b0 < batch; b0 += kPermThreads) {
    const int b = b0 + tid;
    const int c = b < batch ? class_of(table, b) : -1;
    int rank = 0;
#pragma unroll
    for (int k = 0; k < kSlotClasses; ++k) {
      const unsigned m = __ballot_sync(0xffffffffu, c == k);
      if (lane == 0) wcount[warp][k] = __popc(m);
      if (c == k) rank = __popc(m & ((1u << lane) - 1u));
    }
    __syncthreads();
    if (c >= 0) {
      int pos = base[c] + rank;
      for (int w = 0; w < warp; ++w) pos += wcount[w][c];
      perm[pos] = b;
    }
    __syncthreads();                                    // base and wcount read before they change
    if (tid < kSlotClasses) {
      int t = 0;
      for (int w = 0; w < kPermThreads / 32; ++w) t += wcount[w][tid];
      base[tid] += t;
    }
    __syncthreads();
  }
}

static int launch_class_perm(const ProblemParams* table, int batch, int* perm, int* start, cudaStream_t stream) {
  class_perm_kernel<<<1, kPermThreads, 0, stream>>>(table, batch, perm, start);
  AFL_LAUNCH_CHECK("class_perm_kernel");
  return AFL_OK;
}

// Host checks shared by the _dev calls: the per-problem arrays and the status are non-NULL, and the workspace holds
// `need` bytes at a 256-byte boundary.
static int check_dev(const char* who, const int* fs, const int* status, void* ws, size_t ws_bytes, size_t need) {
  if (!fs || !status) { set_error("%s: the per-problem corrupted counts or the status array are NULL", who); return AFL_ERR_BAD_ARG; }
  return check_workspace(who, ws, ws_bytes, need);
}

static int table_dev(const char* rule, int batch, int n, const int* rows, int users_count, const int* ucs,
                     const int* fs, const double* zs, void* ws, size_t ws_bytes, int* status, cudaStream_t stream) {
  const char* who = "afl_batched_table_dev";
  BatchedRule r;
  int rc = parse_rule(who, rule, true, &r);
  if (rc) return rc;
  if (batch < 1 || n < 1) { set_error("%s: batch and n must be >= 1 (got %d, %d)", who, batch, n); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (r == T_ALIE && !zs) { set_error("%s: the per-problem attack strengths are NULL", who); return AFL_ERR_BAD_ARG; }
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch)))) return rc;
  TableArgs a = table_args(r, batch, n, fs, ws, status);
  a.rows = r == T_ALIE ? nullptr : rows; a.ucs = rows ? ucs : nullptr; a.users_count = users_count;
  a.zs = r == T_ALIE ? zs : nullptr;
  return launch_table(a, stream);
}

// afl_defend_batched_dev (max_clients = kBatchMaxClients) and afl_defend_batched_large_dev (kBatchLargeMaxClients):
// afl_defend_batched_rows / _large (rows != NULL) or _each (rows == NULL: n rows and users_count in every problem) with
// device arrays, the same kernels on a device-built table.  Host scalars of those calls become bounds that hold for
// every accepted value: Bulyan's selection width is the caller's sel_ld >= n >= theta_b (the host calls use
// theta_max), and the corrupted counts and users counts that only fill fields a table overrides are passed as 0.
// Above kBatchMaxClients the workspace is the large call's (ProblemParams[batch], perm[batch], then the rule's scratch)
// followed by one kClassStartBytes block for start[]: after each table launch class_perm_kernel groups the problems on
// the device, and the trimmed mean runs one device-count launch per class (tmean::trimmed_mean_classes_dev).  Every
// kernel then reads the table as afl_defend_batched_large does, except the Gram without rows: with n rows in every
// problem its multi-tile centre is the same without the table, and the table of a whole-slot Bulyan holds the second
// stage's tm already.
static int defend_batched_dev(const char* who, int max_clients, const char* rule, const void* G, int batch,
                              int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, const int* rows,
                              int users_count, const int* ucs, const int* fs, float* out, int* idx_out, int* sel_out,
                              int sel_ld, void* ws, size_t ws_bytes, int* status, cudaStream_t stream) {
  BatchedRule r;
  int rc = parse_rule(who, rule, false, &r);
  if (rc || (rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, max_clients))) return rc;
  if (n <= kBatchMaxClients) who = "afl_defend_batched_dev";      // the large call's small form is that call
  if ((rc = check_outputs(who, rule, r, out, idx_out, sel_out))) return rc;
  if (r == B_BULYAN && sel_ld < n) {
    set_error("%s: Bulyan's selection width sel_ld (%d) must be at least n (%d)", who, sel_ld, n);
    return AFL_ERR_BAD_ARG;
  }
  const bool classes = n > kBatchMaxClients, ragged = rows || classes;   // ragged: kernels read rows_b from the table
  const size_t tab_bytes = class_table_bytes(batch, n);
  uint8_t* p = static_cast<uint8_t*>(ws) + tab_bytes;
  const RuleScratch s = rule_scratch(r, batch, n, d, dtype, p);
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, tab_bytes + s.bytes + (classes ? kClassStartBytes : 0)))) return rc;

  TableArgs a = table_args(r, batch, n, fs, ws, status);
  a.rows = rows; a.ucs = rows ? ucs : nullptr; a.users_count = users_count;
  if ((rc = launch_table(a, stream))) return rc;
  const ProblemParams* each = a.table;
  int* perm = reinterpret_cast<int*>(a.table + batch);
  int* start = reinterpret_cast<int*>(p + s.bytes);
  if (r == B_MEAN)
    return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream, ragged ? each : nullptr);
  if (r == B_TM && classes) {
    if ((rc = launch_class_perm(each, batch, perm, start, stream))) return rc;
    return tmean::trimmed_mean_classes_dev(G, n, d, ld, dtype, nullptr, out, batch, batch_stride, 0, d, stream, each,
                                           perm, start);
  }
  if (r == B_TM) return tmean::trimmed_mean_batched(G, n, d, ld, dtype, nullptr, n, 0, out, batch, batch_stride, 0, d, stream, each);
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, s.d2, s.gram, s.gram_bytes, 0, stream,
                            rows ? each : nullptr);
  if (rc) return rc;
  if (r == B_KRUM) return select::krum_from_sqdist(s.d2, n, 0, 0, idx_out, s.sel, s.sel_bytes, stream, batch, each, ragged);
  if ((rc = gram::sqdist_to_dist(s.d2, n, s.dist, stream, batch))) return rc;
  rc = select::bulyan_rounds(s.dist, n, 0, sel_ld, sel_out, s.sel, s.sel_bytes, stream, batch, each, ragged);
  if (rc) return rc;
  a.sel = sel_out; a.sel_ld = sel_ld;                    // second stage's table, and a failed round's status
  if ((rc = launch_table(a, stream))) return rc;
  if (!classes)
    return tmean::trimmed_mean_batched(G, n, d, ld, dtype, sel_out, n, 0, out, batch, batch_stride, sel_ld, d, stream, each);
  if ((rc = launch_class_perm(each, batch, perm, start, stream))) return rc;
  return tmean::trimmed_mean_classes_dev(G, n, d, ld, dtype, sel_out, out, batch, batch_stride, sel_ld, d, stream, each,
                                         perm, start);
}

// afl_alie_batched_each / _large with device arrays; bcast_rows in G's dtype (a 16-bit matrix is written in the kernel).
static int alie_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                            const int* fs, const double* zs, float* mu_out, float* sigma_out, float* crafted_out,
                            void* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* ws, size_t ws_bytes,
                            int* status, cudaStream_t stream) {
  const char* who = "afl_alie_batched_dev";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc) return rc;
  if (!zs) { set_error("%s: the per-problem attack strengths are NULL", who); return AFL_ERR_BAD_ARG; }
  if ((rc = check_bcast(who, bcast_rows, n, d, batch, bcast_batch_stride, bcast_ld))) return rc;
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch)))) return rc;
  TableArgs a = table_args(T_ALIE, batch, n, fs, ws, status);
  a.zs = zs;
  if ((rc = launch_table(a, stream))) return rc;
  return colstats::alie_batched_dev(G, n, d, ld, dtype, mu_out, sigma_out, crafted_out, bcast_rows, bcast_ld, batch,
                                    batch_stride, d, bcast_batch_stride, stream, a.table);
}

// The backdoor crafting's table from device arrays (afl_backdoor_start_batched_dev / _finish_batched_dev):
// backdoor_table's row, with the host calls' count check per problem (f_b < 0 or f_b > n -> AFL_ERR_BAD_ARG, and the
// safe f_b = 0).
static int backdoor_table_dev(const char* who, int batch, int n, const int* fs, const double* zs, const double* lrs,
                              void* ws, size_t ws_bytes, int* status, cudaStream_t stream) {
  if (!zs || !lrs) { set_error("%s: the per-problem attack strengths or learning rates are NULL", who); return AFL_ERR_BAD_ARG; }
  int rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch));
  if (rc) return rc;
  TableArgs a = table_args(T_BACKDOOR, batch, n, fs, ws, status);
  a.zs = zs; a.lrs = lrs;
  return launch_table(a, stream);
}

// afl_backdoor_start_batched with device arrays: n bounds every f_b (the host call's fmax).
static int backdoor_start_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                              const int* fs, const double* zs, const double* lrs, const float* w, int64_t w_batch_stride,
                              float* mu_out, float* sigma_out, float* initial_out, void* ws, size_t ws_bytes,
                              int* status, cudaStream_t stream) {
  const char* who = "afl_backdoor_start_batched_dev";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc || (rc = check_backdoor_start(who, d, w, w_batch_stride, mu_out, sigma_out, initial_out))) return rc;
  if ((rc = backdoor_table_dev(who, batch, n, fs, zs, lrs, ws, ws_bytes, status, stream))) return rc;
  return colstats::backdoor_start(G, n, d, ld, dtype, batch, batch_stride, static_cast<const ProblemParams*>(ws), w,
                                  w_batch_stride, mu_out, sigma_out, initial_out, stream);
}

// afl_backdoor_finish_batched with device arrays; n bounds every f_b, so it also bounds the rows bcast_rows receives.
static int backdoor_finish_dev(int batch, int n, int64_t d, const int* fs, const double* zs, const double* lrs,
                               const float* mu, const float* sigma, const float* initial, const float* mal,
                               int64_t mal_batch_stride, float* crafted_out, float* bcast_rows,
                               int64_t bcast_batch_stride, int64_t bcast_ld, void* ws, size_t ws_bytes, int* status,
                               cudaStream_t stream) {
  const char* who = "afl_backdoor_finish_batched_dev";
  if (!mu || !sigma || !initial || !mal || !crafted_out || d < 1 || n < 1) { set_error("%s: bad argument", who); return AFL_ERR_BAD_ARG; }
  int rc = check_backdoor_finish(who, batch, d, mal_batch_stride);
  if (rc || (rc = check_bcast(who, bcast_rows, n, d, batch, bcast_batch_stride, bcast_ld))) return rc;
  if ((rc = backdoor_table_dev(who, batch, n, fs, zs, lrs, ws, ws_bytes, status, stream))) return rc;
  return colstats::backdoor_finish(batch, d, static_cast<const ProblemParams*>(ws), mu, sigma, initial, mal,
                                   mal_batch_stride, crafted_out, bcast_rows, bcast_batch_stride, bcast_ld, stream);
}

// afl_attack_metrics_batched_rows (rows != NULL) or _each with device arrays.
static int attack_metrics_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                              const int* rows, const int* fs, const float* agg, const int* idx, const int* sel,
                              int sel_ld, float* dev_out, double* sums_out, float* honest_out, int* krum_hit,
                              int* mal_count, int* sel_count, void* ws, size_t ws_bytes, int* status,
                              cudaStream_t stream) {
  const char* who = "afl_attack_metrics_batched_dev";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc || (rc = check_metrics_inputs(who, agg, idx, sel, sel_ld, dev_out, sums_out, krum_hit, mal_count, sel_count)))
    return rc;
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch) + metrics_partial_bytes(batch, d, dtype)))) return rc;
  TableArgs a = table_args(T_METRICS, batch, n, fs, ws, status);
  a.rows = rows;
  if ((rc = launch_table(a, stream))) return rc;
  return colstats::attack_metrics(G, batch, batch_stride, n, d, ld, dtype, 0, a.table, agg, idx, sel, sel_ld, dev_out,
                                  sums_out, honest_out, krum_hit, mal_count, sel_count,
                                  static_cast<uint8_t*>(ws) + table_bytes(batch), stream, rows != nullptr);
}

// afl_attack_trace_dev's workspace: the T_METRICS table, then double[batch][tiles][3] partial sums.
static size_t trace_workspace_bytes(int batch, int64_t d) {
  return table_bytes(batch) +
         align_up(static_cast<size_t>(batch) * colstats::deviation_tiles(d, AFL_F32) * 3 * sizeof(double), 256);
}

// One epoch's attack figures of an fp32 batch into row *slot of caller-held tables: afl_attack_metrics_batched_dev's
// table and selection checks, then colstats::attack_trace.
static int attack_trace_dev(const float* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                            const int* rows, const int* fs, const float* agg, const int* idx, const int* sel,
                            int sel_ld, const int* slot, int n_slots, int64_t table_ld, float* agg_dev,
                            float* mal_dev, int* idx_out, int* mal_count, int* sel_count, void* ws, size_t ws_bytes,
                            int* status, cudaStream_t stream) {
  const char* who = "afl_attack_trace_dev";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, AFL_F32, INT32_MAX);
  if (rc) return rc;
  if (!agg || !slot) { set_error("%s: the aggregate agg and the device slot are required (NULL given)", who); return AFL_ERR_BAD_ARG; }
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  if (table_ld < batch) {
    set_error("%s: table_ld %lld is less than batch %d", who, static_cast<long long>(table_ld), batch);
    return AFL_ERR_BAD_ARG;
  }
  if ((rc = check_sel(who, sel, sel_ld, mal_count, sel_count))) return rc;
  if (idx_out && !idx) { set_error("%s: idx_out needs idx", who); return AFL_ERR_BAD_ARG; }
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, trace_workspace_bytes(batch, d)))) return rc;
  TableArgs a = table_args(T_METRICS, batch, n, fs, ws, status);
  a.rows = rows;
  if ((rc = launch_table(a, stream))) return rc;
  return colstats::attack_trace(G, batch, batch_stride, n, d, ld, a.table, agg, idx, sel, sel_ld, slot, n_slots,
                                table_ld, agg_dev, mal_dev, idx_out, mal_count, sel_count,
                                static_cast<uint8_t*>(ws) + table_bytes(batch), stream, rows != nullptr);
}

}  // namespace afl

using namespace afl;

extern "C" {

const char* afl_version(void) { return "afl_b200 0.1.0 (sm_90a)"; }
const char* afl_last_error(void) { return g_err; }
uint64_t afl_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int afl_device_info(int* sms, int* cc_major, int* cc_minor, size_t* free_bytes, size_t* total_bytes) {
  int dev = 0;
  AFL_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  AFL_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sms) *sms = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  size_t f = 0, t = 0;
  AFL_CUDA(cudaMemGetInfo(&f, &t));
  if (free_bytes) *free_bytes = f;
  if (total_bytes) *total_bytes = t;
  return AFL_OK;
}

int afl_profile_enable(int on) { g_prof_on.store(on == 2 ? 2 : (on ? 1 : 0)); return AFL_OK; }
int afl_profile_read(const char* kernel, double* total_ms, int* launches) {
  if (!kernel) { set_error("afl_profile_read: kernel is NULL"); return AFL_ERR_BAD_ARG; }
  return profile_read(kernel, total_ms, launches);
}

int afl_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, void* stream) {
  return colstats::mean(G, n, d, ld, dtype, out, static_cast<cudaStream_t>(stream));
}

size_t afl_sqdist_workspace_bytes(int n, int64_t d, int dtype, int flags) {
  if (n < 1 || d < 1) return 256;
  return gram::workspace_bytes(n, d, dtype, flags);
}
int afl_sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out, void* workspace,
                       size_t workspace_bytes, int flags, void* stream) {
  return gram::sqdist_partial(G, n, d, ld, dtype, d2_out, workspace, workspace_bytes, flags,
                              static_cast<cudaStream_t>(stream));
}
int afl_sqdist_to_dist(const double* d2, int n, float* dist, void* stream) {
  return gram::sqdist_to_dist(d2, n, dist, static_cast<cudaStream_t>(stream));
}

size_t afl_select_workspace_bytes(int n) { return select::workspace_bytes(n); }
int afl_krum_select(const float* dist, int n, int users_count, int corrupted_count, int* idx_out, float* scores_out,
                    void* workspace, size_t workspace_bytes, void* stream) {
  return select::krum_select(dist, n, users_count, corrupted_count, idx_out, scores_out, workspace, workspace_bytes,
                             static_cast<cudaStream_t>(stream));
}
int afl_krum_from_sqdist(const double* d2, int n, int users_count, int corrupted_count, int* idx_out, void* workspace,
                         size_t workspace_bytes, void* stream) {
  return select::krum_from_sqdist(d2, n, users_count, corrupted_count, idx_out, workspace, workspace_bytes,
                                  static_cast<cudaStream_t>(stream));
}
int afl_bulyan_select(const float* dist, int n, int users_count, int corrupted_count, int* sel_out, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return select::bulyan_select(dist, n, users_count, corrupted_count, sel_out, workspace, workspace_bytes,
                               static_cast<cudaStream_t>(stream));
}

int afl_trimmed_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                     int corrupted_count, float* out, void* stream) {
  return tmean::trimmed_mean(G, n, d, ld, dtype, row_index, n_rows, corrupted_count, out,
                             static_cast<cudaStream_t>(stream));
}


int afl_gather_row(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* idx_dev, float* out,
                   void* stream) {
  return colstats::gather_row(G, n, d, ld, dtype, idx_dev, out, static_cast<cudaStream_t>(stream));
}

int afl_alie(const void* G_mal, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
             float* crafted_out, float* bcast_rows, int64_t bcast_ld, void* stream) {
  return colstats::alie(G_mal, f, d, ld, dtype, z, mu_out, sigma_out, crafted_out, bcast_rows, bcast_ld,
                        static_cast<cudaStream_t>(stream));
}

int afl_alie_band(const float* mu, const float* sigma, double z, const float* x, float* out, int64_t d, void* stream) {
  return colstats::alie_band(mu, sigma, z, x, out, d, static_cast<cudaStream_t>(stream));
}

int afl_momentum_step(float* weights, float* velocity, const float* grads, int64_t d, float momentum,
                      float learning_rate, void* stream) {
  return colstats::momentum_step(weights, velocity, grads, d, momentum, learning_rate,
                                 static_cast<cudaStream_t>(stream));
}

int afl_momentum_step_batched(float* weights, float* velocity, const float* grads, int batch, int64_t d,
                              float momentum, const float* learning_rate, void* stream) {
  return colstats::momentum_step_batched(weights, velocity, grads, batch, d, momentum, learning_rate,
                                         static_cast<cudaStream_t>(stream));
}

int afl_defend_host(const char* rule, const float* G_host, int n, int64_t d, int64_t ld, int users_count,
                    int corrupted_count, float* out_host, int* idx_out, int64_t slab_cols) {
  if (!rule) { set_error("afl_defend_host: rule is NULL"); return AFL_ERR_BAD_ARG; }
  return defend_host(rule, G_host, n, d, ld, users_count, corrupted_count, out_host, idx_out, slab_cols);
}

int afl_sqdist_host(const float* G_host, int n, int64_t d, int64_t ld, double* d2_out, int64_t slab_cols) {
  return sqdist_host(G_host, n, d, ld, d2_out, slab_cols);
}

int afl_bulyan_host(const float* G_host, int n, int64_t d, int64_t ld, int users_count, int corrupted_count,
                    float* out_host, int* sel_host, int64_t slab_cols) {
  return bulyan_host("afl_bulyan_host", G_host, n, d, ld, users_count, corrupted_count, out_host, sel_host, slab_cols);
}

int afl_alie_host(const float* const* rows, int f, int64_t d, double z, float* mu_out, float* sigma_out,
                  float* crafted_out, int64_t slab_cols) {
  return alie_host(rows, f, d, z, mu_out, sigma_out, crafted_out, slab_cols);
}

size_t afl_batched_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD || batch < 1 || batch > kBatchMax || n < 1 || n > kBatchMaxClients || d < 1) return 0;
  if (r == B_MEAN || r == B_TM) return 256;
  return rule_scratch(r, batch, n, d, dtype).bytes;
}

size_t afl_batched_each_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const bool alie = rule && !strcmp(rule, "ALIE");
  const BatchedRule r = batched_rule(rule);
  if ((r == B_BAD && !alie) || batch < 1 || batch > kBatchMax || n < 1 || n > kBatchMaxClients || d < 1) return 0;
  return table_bytes(batch) + rule_scratch(r, batch, n, d, dtype).bytes;
}

int afl_defend_batched(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                       int dtype, int users_count, int corrupted_count, float* out, int* idx_out, int* sel_out,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return defend_batched("afl_defend_batched", kBatchMaxClients, false, rule, G, batch, batch_stride, n, d, ld, dtype,
                        nullptr, nullptr, users_count, nullptr, corrupted_count, out, idx_out, sel_out, workspace,
                        workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_defend_batched_each(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                            int64_t ld, int dtype, int users_count, const int* corrupted_counts, float* out, int* idx_out,
                            int* sel_out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!corrupted_counts) {
    set_error("afl_defend_batched_each: the per-problem corrupted counts are NULL");
    return AFL_ERR_BAD_ARG;
  }
  return defend_batched("afl_defend_batched_each", kBatchMaxClients, false, rule, G, batch, batch_stride, n, d, ld, dtype,
                        nullptr, nullptr, users_count, corrupted_counts, 0, out, idx_out, sel_out, workspace,
                        workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_alie_batched(const void* G_mal, int batch, int64_t batch_stride, int f, int64_t d, int64_t ld, int dtype, double z,
                     float* mu_out, float* sigma_out, float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride,
                     int64_t bcast_ld, void* stream) {
  return alie_batched("afl_alie_batched", G_mal, batch, batch_stride, f, d, ld, dtype, f, z, nullptr, nullptr, mu_out,
                      sigma_out, crafted_out, bcast_rows, bcast_batch_stride, bcast_ld, nullptr, 0,
                      static_cast<cudaStream_t>(stream));
}

int afl_alie_batched_each(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                          const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                          float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!f) { set_error("afl_alie_batched_each: the per-problem corrupted counts are NULL"); return AFL_ERR_BAD_ARG; }
  return alie_batched("afl_alie_batched_each", G, batch, batch_stride, n, d, ld, dtype, 0, 0.0, f, z, mu_out, sigma_out,
                      crafted_out, bcast_rows, bcast_batch_stride, bcast_ld, workspace, workspace_bytes,
                      static_cast<cudaStream_t>(stream));
}

size_t afl_batched_rows_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  if (batched_rule(rule) == B_BAD) return 0;
  return afl_batched_each_workspace_bytes(rule, batch, n, d, dtype);
}

int afl_defend_batched_rows(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                            int64_t ld, int dtype, const int* rows, const int* users_counts, const int* corrupted_counts,
                            float* out, int* idx_out, int* sel_out, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return defend_batched("afl_defend_batched_rows", kBatchMaxClients, true, rule, G, batch, batch_stride, n, d, ld, dtype,
                        rows, users_counts, 0, corrupted_counts, 0, out, idx_out, sel_out, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream));
}

size_t afl_batched_large_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD || n < 1 || n > kBatchLargeMaxClients) return 0;
  if (n <= kBatchMaxClients) return afl_batched_rows_workspace_bytes(rule, batch, n, d, dtype);
  if (batch < 1 || batch > kBatchMax || d < 1 || (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16)) return 0;
  return class_table_bytes(batch, n) + rule_scratch(r, batch, n, d, dtype).bytes;
}

int afl_defend_batched_large(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                             int64_t ld, int dtype, const int* rows, const int* users_counts,
                             const int* corrupted_counts, float* out, int* idx_out, int* sel_out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  std::vector<int> all;                                 // rows == NULL: n rows in every problem
  if (!rows && batch >= 1 && batch <= kBatchMax) {
    all.assign(static_cast<size_t>(batch), n);
    rows = all.data();
  }
  return defend_batched("afl_defend_batched_large", kBatchLargeMaxClients, true, rule, G, batch, batch_stride, n, d, ld,
                        dtype, rows, users_counts, 0, corrupted_counts, 0, out, idx_out, sel_out, workspace,
                        workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_alie_batched_large(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                           const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                           float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                           size_t workspace_bytes, void* stream) {
  if (!f) { set_error("afl_alie_batched_large: the per-problem corrupted counts are NULL"); return AFL_ERR_BAD_ARG; }
  return alie_batched("afl_alie_batched_large", G, batch, batch_stride, n, d, ld, dtype, 0, 0.0, f, z, mu_out, sigma_out,
                      crafted_out, bcast_rows, bcast_batch_stride, bcast_ld, workspace, workspace_bytes,
                      static_cast<cudaStream_t>(stream), INT32_MAX);
}

size_t afl_metrics_workspace_bytes(int batch, int n, int64_t d, int dtype) {
  if (batch < 1 || batch > kBatchMax || n < 1 || d < 1 || (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16)) return 0;
  return table_bytes(batch) + metrics_partial_bytes(batch, d, dtype);
}

int afl_attack_metrics_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                               int corrupted_count, const float* agg, const int* idx, const int* sel, int sel_ld,
                               float* dev_out, double* sums_out, float* honest_out, int* krum_hit, int* mal_count,
                               int* sel_count, void* workspace, size_t workspace_bytes, void* stream) {
  return attack_metrics(G, batch, batch_stride, n, d, ld, dtype, corrupted_count, nullptr, agg, idx, sel, sel_ld, dev_out,
                        sums_out, honest_out, krum_hit, mal_count, sel_count, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream));
}

int afl_attack_metrics_batched_each(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                    int dtype, const int* corrupted_counts, const float* agg, const int* idx,
                                    const int* sel, int sel_ld, float* dev_out, double* sums_out, float* honest_out,
                                    int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!corrupted_counts) {
    set_error("afl_attack_metrics_batched_each: the per-problem corrupted counts are NULL");
    return AFL_ERR_BAD_ARG;
  }
  return attack_metrics(G, batch, batch_stride, n, d, ld, dtype, 0, corrupted_counts, agg, idx, sel, sel_ld, dev_out,
                        sums_out, honest_out, krum_hit, mal_count, sel_count, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream));
}

int afl_attack_metrics_batched_rows(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                    int dtype, const int* rows, const int* corrupted_counts, const float* agg,
                                    const int* idx, const int* sel, int sel_ld, float* dev_out, double* sums_out,
                                    float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  if (!rows || !corrupted_counts) {
    set_error("afl_attack_metrics_batched_rows: the per-problem row counts or corrupted counts are NULL");
    return AFL_ERR_BAD_ARG;
  }
  return attack_metrics(G, batch, batch_stride, n, d, ld, dtype, 0, corrupted_counts, agg, idx, sel, sel_ld, dev_out,
                        sums_out, honest_out, krum_hit, mal_count, sel_count, workspace, workspace_bytes,
                        static_cast<cudaStream_t>(stream), rows);
}

int afl_backdoor_start_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                               const int* f, const double* z, const double* lr, const float* w, int64_t w_batch_stride,
                               float* mu_out, float* sigma_out, float* initial_out, void* workspace,
                               size_t workspace_bytes, void* stream) {
  return backdoor_start(G, batch, batch_stride, n, d, ld, dtype, f, z, lr, w, w_batch_stride, mu_out, sigma_out,
                        initial_out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_backdoor_finish_batched(int batch, int64_t d, const int* f, const double* z, const double* lr, const float* mu,
                                const float* sigma, const float* initial, const float* mal, int64_t mal_batch_stride,
                                float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld,
                                void* workspace, size_t workspace_bytes, void* stream) {
  return backdoor_finish(batch, d, f, z, lr, mu, sigma, initial, mal, mal_batch_stride, crafted_out, bcast_rows,
                         bcast_batch_stride, bcast_ld, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_batched_table_dev(const char* rule, int batch, int n, const int* rows, int users_count, const int* users_counts,
                          const int* corrupted_counts, const double* z, void* workspace, size_t workspace_bytes,
                          int* status, void* stream) {
  return table_dev(rule, batch, n, rows, users_count, users_counts, corrupted_counts, z, workspace, workspace_bytes,
                   status, static_cast<cudaStream_t>(stream));
}

int afl_defend_batched_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                           int dtype, const int* rows, int users_count, const int* users_counts,
                           const int* corrupted_counts, float* out, int* idx_out, int* sel_out, int sel_ld,
                           void* workspace, size_t workspace_bytes, int* status, void* stream) {
  return defend_batched_dev("afl_defend_batched_dev", kBatchMaxClients, rule, G, batch, batch_stride, n, d, ld, dtype,
                            rows, users_count, users_counts, corrupted_counts, out, idx_out, sel_out, sel_ld, workspace,
                            workspace_bytes, status, static_cast<cudaStream_t>(stream));
}

size_t afl_batched_large_dev_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const size_t large = afl_batched_large_workspace_bytes(rule, batch, n, d, dtype);
  if (!large || n <= kBatchMaxClients) return large;
  return large + kClassStartBytes;
}

int afl_defend_batched_large_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                                 int64_t ld, int dtype, const int* rows, int users_count, const int* users_counts,
                                 const int* corrupted_counts, float* out, int* idx_out, int* sel_out, int sel_ld,
                                 void* workspace, size_t workspace_bytes, int* status, void* stream) {
  return defend_batched_dev("afl_defend_batched_large_dev", kBatchLargeMaxClients, rule, G, batch, batch_stride, n, d,
                            ld, dtype, rows, users_count, users_counts, corrupted_counts, out, idx_out, sel_out, sel_ld,
                            workspace, workspace_bytes, status, static_cast<cudaStream_t>(stream));
}

int afl_alie_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                         const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                         void* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                         size_t workspace_bytes, int* status, void* stream) {
  return alie_batched_dev(G, batch, batch_stride, n, d, ld, dtype, f, z, mu_out, sigma_out, crafted_out, bcast_rows,
                          bcast_batch_stride, bcast_ld, workspace, workspace_bytes, status,
                          static_cast<cudaStream_t>(stream));
}

int afl_attack_metrics_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                   int dtype, const int* rows, const int* corrupted_counts, const float* agg,
                                   const int* idx, const int* sel, int sel_ld, float* dev_out, double* sums_out,
                                   float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                   size_t workspace_bytes, int* status, void* stream) {
  return attack_metrics_dev(G, batch, batch_stride, n, d, ld, dtype, rows, corrupted_counts, agg, idx, sel, sel_ld,
                            dev_out, sums_out, honest_out, krum_hit, mal_count, sel_count, workspace, workspace_bytes,
                            status, static_cast<cudaStream_t>(stream));
}

size_t afl_attack_trace_workspace_bytes(int batch, int64_t d) {
  if (batch < 1 || batch > kBatchMax || d < 1) return 0;
  return trace_workspace_bytes(batch, d);
}

int afl_attack_trace_dev(const float* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, const int* rows,
                         const int* corrupted_counts, const float* agg, const int* idx, const int* sel, int sel_ld,
                         const int* slot, int n_slots, int64_t table_ld, float* agg_dev, float* mal_dev, int* idx_out,
                         int* mal_count, int* sel_count, void* workspace, size_t workspace_bytes, int* status,
                         void* stream) {
  return attack_trace_dev(G, batch, batch_stride, n, d, ld, rows, corrupted_counts, agg, idx, sel, sel_ld, slot,
                          n_slots, table_ld, agg_dev, mal_dev, idx_out, mal_count, sel_count, workspace,
                          workspace_bytes, status, static_cast<cudaStream_t>(stream));
}

int afl_backdoor_start_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                   int dtype, const int* f, const double* z, const double* lr, const float* w,
                                   int64_t w_batch_stride, float* mu_out, float* sigma_out, float* initial_out,
                                   void* workspace, size_t workspace_bytes, int* status, void* stream) {
  return backdoor_start_dev(G, batch, batch_stride, n, d, ld, dtype, f, z, lr, w, w_batch_stride, mu_out, sigma_out,
                            initial_out, workspace, workspace_bytes, status, static_cast<cudaStream_t>(stream));
}

int afl_backdoor_finish_batched_dev(int batch, int n, int64_t d, const int* f, const double* z, const double* lr,
                                    const float* mu, const float* sigma, const float* initial, const float* mal,
                                    int64_t mal_batch_stride, float* crafted_out, float* bcast_rows,
                                    int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                                    size_t workspace_bytes, int* status, void* stream) {
  return backdoor_finish_dev(batch, n, d, f, z, lr, mu, sigma, initial, mal, mal_batch_stride, crafted_out, bcast_rows,
                             bcast_batch_stride, bcast_ld, workspace, workspace_bytes, status,
                             static_cast<cudaStream_t>(stream));
}

}  // extern "C"
