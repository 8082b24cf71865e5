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
// ProblemParams row per problem, built here with the single call's own host code (krum_take, tmean::shape) and copied
// to the start of the workspace; the scalar call's layout follows it.  The scalar calls pass no table and run as they
// always have.
// The large calls (afl_defend_batched_large) take up to 1024 clients per problem: every Gram form is batched for any
// tile count, and the register-resident trimmed-mean kernels end at 1024 rows.
// ------------------------------------------------------------------------------------------------
constexpr int kBatchMaxClients = 128;            // one Gram tile
constexpr int kBatchLargeMaxClients = 1024;      // the largest register-resident trimmed-mean kernel (S = 32)
constexpr int kBatchMax = 65535;                 // grid y / z limit

enum BatchedRule { B_BAD, B_MEAN, B_KRUM, B_TM, B_BULYAN };
static BatchedRule batched_rule(const char* rule) {
  if (!rule) return B_BAD;
  if (!strcmp(rule, "NoDefense")) return B_MEAN;
  if (!strcmp(rule, "Krum")) return B_KRUM;
  if (!strcmp(rule, "TrimmedMean")) return B_TM;
  if (!strcmp(rule, "Bulyan")) return B_BULYAN;
  return B_BAD;
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

static size_t table_bytes(int batch) { return align_up(static_cast<size_t>(batch) * sizeof(ProblemParams), 256); }
// The table of a batch with more than kBatchMaxClients rows per slot: ProblemParams[batch], then int perm[batch], the
// problems grouped by trimmed-mean slot class (tmean::trimmed_mean_classes).
static size_t class_table_bytes(int batch, int n) {
  if (n <= kBatchMaxClients) return table_bytes(batch);
  return align_up(static_cast<size_t>(batch) * (sizeof(ProblemParams) + sizeof(int)), 256);
}

// The rule's scratch after the table (0: the rule needs none).
static size_t batched_ws_parts(BatchedRule r, int batch, int n, int64_t d, int dtype, size_t* gram_ws, size_t* tabs) {
  *gram_ws = 0; *tabs = 0;
  if (r != B_KRUM && r != B_BULYAN) return 0;
  const size_t nn = static_cast<size_t>(batch) * n * n;
  *gram_ws = align_up(gram::workspace_bytes(n, d, dtype, 0, batch), 256);
  *tabs = align_up(nn * 8, 256) + (r == B_BULYAN ? align_up(nn * 4, 256) : 0);
  return *gram_ws + *tabs + select::workspace_bytes(n, batch);
}

// Workspace check, then the table built by `row(b, ProblemParams&)` copied to the workspace start (pageable source:
// the copy has taken the values when cudaMemcpyAsync returns).  Returns the device table in *table.
template <typename Row>
static int upload_table(const char* who, int batch, void* ws, size_t ws_bytes, size_t need, cudaStream_t stream,
                        Row row, const ProblemParams** table) {
  if (!ws || ws_bytes < need || reinterpret_cast<uintptr_t>(ws) % 256 != 0) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  std::vector<ProblemParams> host(static_cast<size_t>(batch));
  for (int b = 0; b < batch; ++b) row(b, host[b]);
  AFL_CUDA(cudaMemcpyAsync(ws, host.data(), host.size() * sizeof(ProblemParams), cudaMemcpyHostToDevice, stream));
  *table = static_cast<const ProblemParams*>(ws);
  return AFL_OK;
}

// upload_table followed by the problems grouped by the trimmed-mean slot class of their tm.n_rows, in one copy: the
// device permutation in *perm, the class sizes in counts[kSlotClasses] (host).
template <typename Row>
static int upload_class_table(const char* who, int batch, void* ws, size_t ws_bytes, size_t need, cudaStream_t stream,
                              Row row, const ProblemParams** table, const int** perm, int* counts) {
  if (!ws || ws_bytes < need || reinterpret_cast<uintptr_t>(ws) % 256 != 0) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  const size_t nb = static_cast<size_t>(batch);
  std::vector<ProblemParams> host(nb);
  std::vector<int> cls(nb), order(nb);
  for (int c = 0; c < kSlotClasses; ++c) counts[c] = 0;
  for (int b = 0; b < batch; ++b) {
    row(b, host[b]);
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
  *table = static_cast<const ProblemParams*>(ws);
  *perm = reinterpret_cast<const int*>(static_cast<const uint8_t*>(ws) + nb * sizeof(ProblemParams));
  return AFL_OK;
}

// fs == NULL: every problem has corrupted_count f (afl_defend_batched).  Otherwise problem b has fs[b]
// (afl_defend_batched_each): f is unused, the preconditions hold per problem, and the workspace starts with the table.
static int defend_batched(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                          int dtype, int users_count, int f, const int* fs, float* out, int* idx_out, int* sel_out,
                          void* ws, size_t ws_bytes, cudaStream_t stream) {
  const char* who = fs ? "afl_defend_batched_each" : "afl_defend_batched";
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD) { set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)"); return AFL_ERR_BAD_ARG; }
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype);
  if (rc) return rc;
  int fmin = f, fmax = f;
  if (fs && (rc = check_counts(who, fs, batch, INT32_MAX / 4, &fmin, &fmax))) return rc;
  if ((r != B_KRUM && !out) || (r == B_KRUM && !idx_out) || (r == B_BULYAN && !sel_out) || fmin < 0) {
    set_error("%s: %s needs %s", who, rule, r == B_KRUM ? "idx_out" : r == B_BULYAN ? "out and sel_out" : "out");
    return AFL_ERR_BAD_ARG;
  }
  // the reference's asserts (defences.py:24-25, 56), per problem
  const int need_f = r == B_KRUM ? 2 * fmax + 1 : r == B_BULYAN ? 4 * fmax + 3 : 0;
  if (users_count < need_f) {
    const char* what = r == B_KRUM ? "krum: users_count >= 2*corrupted_count + 1" : "bulyan: users_count >= 4*corrupted_count + 3";
    int b = 0;
    while (fs && fs[b] != fmax) ++b;
    if (fs) set_error("%s violated (%d, %d) in problem %d", what, users_count, fmax, b);
    else set_error("%s violated (%d, %d)", what, users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if (r == B_BULYAN && users_count != n) {
    set_error("%s: Bulyan's users_count (%d) must equal the number of rows (%d)", who, users_count, n);
    return AFL_ERR_UNSUPPORTED;
  }
  size_t gram_ws = 0, tabs = 0;
  const size_t rule_ws = batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
  const ProblemParams* each = nullptr;
  uint8_t* p = static_cast<uint8_t*>(ws);
  if (fs && r != B_MEAN) {                              // NoDefense ignores f, as the reference does
    rc = upload_table(who, batch, ws, ws_bytes, table_bytes(batch) + rule_ws, stream, [&](int b, ProblemParams& q) {
      q.f = fs[b];
      q.take = select::krum_take(n, users_count, fs[b]);
      q.theta = users_count - 2 * fs[b];
      q.tm = r == B_BULYAN ? tmean::shape(q.theta, 2 * fs[b]) : tmean::shape(n, fs[b]);
    }, &each);
    if (rc) return rc;
    p += table_bytes(batch);
    ws_bytes -= table_bytes(batch);
  }
  if (r == B_MEAN) return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream);
  if (r == B_TM)
    return tmean::trimmed_mean_batched(G, n, d, ld, dtype, nullptr, n, fmin, out, batch, batch_stride, 0, d, stream, each);
  if (ws_bytes < rule_ws || !p || reinterpret_cast<uintptr_t>(p) % 256 != 0) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, rule_ws);
    return AFL_ERR_WORKSPACE;
  }
  const size_t nn = static_cast<size_t>(batch) * n * n;
  double* d2 = reinterpret_cast<double*>(p);
  float* dist = reinterpret_cast<float*>(p + align_up(nn * 8, 256));
  void* sel_ws = p + tabs + gram_ws;
  const size_t sel_ws_bytes = ws_bytes - tabs - gram_ws;
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, d2, p + tabs, gram_ws, 0, stream);
  if (rc) return rc;
  if (r == B_KRUM)
    return select::krum_from_sqdist(d2, n, users_count, fmin, idx_out, sel_ws, sel_ws_bytes, stream, batch, each);
  const int theta = users_count - 2 * fmin;             // the row length of sel_out
  rc = gram::sqdist_to_dist(d2, n, dist, stream, batch); if (rc) return rc;
  rc = select::bulyan_select(dist, n, users_count, fmin, sel_out, sel_ws, sel_ws_bytes, stream, batch, each);
  if (rc) return rc;
  return tmean::trimmed_mean_batched(G, n, d, ld, dtype, sel_out, theta, 2 * fmin, out, batch, batch_stride, theta, d,
                                     stream, each);
}

// A ragged batch (afl_defend_batched_rows): problem b is rows 0..rows[b]-1 of its n-row slot, with its own users_count
// ucs[b] and corrupted count fs[b].  Every check is the single call's, per problem and before any CUDA call; the table
// rows come from the single call's host helpers on (rows[b], ucs[b], fs[b]), and each kernel reads the problem's row
// count from them: tm.n_rows (the Gram centre, Krum, TrimmedMean, NoDefense), theta + 2f (Bulyan's selection, whose
// users_count is its row count).  Bulyan's second stage needs tm = shape(theta, 2f): that table is copied over the
// first one after the selection kernels, in stream order.  The workspace layout is afl_defend_batched_each's.
// max_clients: kBatchMaxClients (afl_defend_batched_rows) or kBatchLargeMaxClients (afl_defend_batched_large).  Slots of
// more than kBatchMaxClients rows append the problems' trimmed-mean class permutation to the table
// (class_table_bytes), and the trimmed mean runs one launch per class (tmean::trimmed_mean_classes).
static int defend_batched_rows(const char* who, int max_clients, const char* rule, const void* G, int batch,
                               int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, const int* rows,
                               const int* ucs, const int* fs, float* out, int* idx_out, int* sel_out, void* ws,
                               size_t ws_bytes, cudaStream_t stream) {
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD) { set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)"); return AFL_ERR_BAD_ARG; }
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, max_clients);
  if (rc) return rc;
  if (!rows || !ucs) { set_error("%s: the per-problem row counts or users counts are NULL", who); return AFL_ERR_BAD_ARG; }
  int fmin = 0, fmax = 0;
  if ((rc = check_counts(who, fs, batch, INT32_MAX / 4, &fmin, &fmax))) return rc;
  for (int b = 0; b < batch; ++b)
    if (rows[b] < 1 || rows[b] > n) {
      set_error("%s: row count %d of problem %d is outside [1, %d]", who, rows[b], b, n);
      return AFL_ERR_BAD_ARG;
    }
  if ((r != B_KRUM && !out) || (r == B_KRUM && !idx_out) || (r == B_BULYAN && !sel_out)) {
    set_error("%s: %s needs %s", who, rule, r == B_KRUM ? "idx_out" : r == B_BULYAN ? "out and sel_out" : "out");
    return AFL_ERR_BAD_ARG;
  }
  int theta_max = 0;
  for (int b = 0; b < batch; ++b) {
    // the reference's asserts (defences.py:24-25, 56), per problem
    const int64_t need = r == B_KRUM ? 2 * static_cast<int64_t>(fs[b]) + 1 : r == B_BULYAN ? 4 * static_cast<int64_t>(fs[b]) + 3 : 0;
    if (ucs[b] < need) {
      set_error("%s violated (%d, %d) in problem %d",
                r == B_KRUM ? "krum: users_count >= 2*corrupted_count + 1" : "bulyan: users_count >= 4*corrupted_count + 3",
                ucs[b], fs[b], b);
      return AFL_ERR_PRECONDITION;
    }
    if (r == B_BULYAN && ucs[b] != rows[b]) {
      set_error("%s: Bulyan's users_count (%d) must equal the number of rows (%d) in problem %d", who, ucs[b], rows[b], b);
      return AFL_ERR_UNSUPPORTED;
    }
    const int theta = ucs[b] - 2 * fs[b];
    theta_max = theta > theta_max ? theta : theta_max;
  }
  size_t gram_ws = 0, tabs = 0;
  const size_t rule_ws = batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
  const bool classes = n > kBatchMaxClients;
  const size_t tab_bytes = class_table_bytes(batch, n);
  const ProblemParams* each = nullptr;
  const int* perm = nullptr;
  int counts[kSlotClasses];
  auto row = [&](int b, ProblemParams& q) {
    q.f = fs[b];
    q.take = select::krum_take(rows[b], ucs[b], fs[b]);
    q.theta = ucs[b] - 2 * fs[b];
    q.tm = tmean::shape(rows[b], fs[b]);
  };
  rc = classes ? upload_class_table(who, batch, ws, ws_bytes, tab_bytes + rule_ws, stream, row, &each, &perm, counts)
               : upload_table(who, batch, ws, ws_bytes, tab_bytes + rule_ws, stream, row, &each);
  if (rc) return rc;
  uint8_t* p = static_cast<uint8_t*>(ws) + tab_bytes;
  if (r == B_MEAN) return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream, each);
  if (r == B_TM && classes)
    return tmean::trimmed_mean_classes(G, n, d, ld, dtype, nullptr, out, batch, batch_stride, 0, d, stream, each, perm,
                                       counts);
  if (r == B_TM)
    return tmean::trimmed_mean_batched(G, n, d, ld, dtype, nullptr, n, fmin, out, batch, batch_stride, 0, d, stream, each);
  const size_t nn = static_cast<size_t>(batch) * n * n;
  double* d2 = reinterpret_cast<double*>(p);
  float* dist = reinterpret_cast<float*>(p + align_up(nn * 8, 256));
  void* sel_ws = p + tabs + gram_ws;
  const size_t sel_ws_bytes = ws_bytes - tab_bytes - tabs - gram_ws;
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, d2, p + tabs, gram_ws, 0, stream, each);
  if (rc) return rc;
  if (r == B_KRUM)
    return select::krum_from_sqdist(d2, n, 0, 0, idx_out, sel_ws, sel_ws_bytes, stream, batch, each, true);
  rc = gram::sqdist_to_dist(d2, n, dist, stream, batch); if (rc) return rc;
  rc = select::bulyan_rounds(dist, n, fmin, theta_max, sel_out, sel_ws, sel_ws_bytes, stream, batch, each, true);
  if (rc) return rc;
  auto row2 = [&](int b, ProblemParams& q) {
    row(b, q);
    q.tm = tmean::shape(q.theta, 2 * fs[b]);              // the trimmed mean of the theta_b selected rows with 2 f_b
  };
  if (classes) {
    rc = upload_class_table(who, batch, ws, ws_bytes, tab_bytes + rule_ws, stream, row2, &each, &perm, counts);
    if (rc) return rc;
    return tmean::trimmed_mean_classes(G, n, d, ld, dtype, sel_out, out, batch, batch_stride, theta_max, d, stream, each,
                                       perm, counts);
  }
  rc = upload_table(who, batch, ws, ws_bytes, tab_bytes + rule_ws, stream, row2, &each);
  if (rc) return rc;
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
  if (bcast_rows && fmax > 0 &&
      (bcast_ld < d || (batch > 1 && bcast_batch_stride < static_cast<int64_t>(fmax - 1) * bcast_ld + d))) {
    set_error("%s: bcast_ld / bcast_batch_stride make the written rows overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  const ProblemParams* each = nullptr;
  if (fs) {
    rc = upload_table(who, batch, ws, ws_bytes, table_bytes(batch), stream, [&](int b, ProblemParams& q) {
      q.f = fs[b];
      q.z = static_cast<float>(zs[b]);
      q.write = fs[b] > 0 && zs[b] != 0.0;             // malicious.py:20-21: z == 0 computes the statistics only
    }, &each);
    if (rc) return rc;
  }
  return colstats::alie_batched(G, fmax, d, ld, dtype, z, mu_out, sigma_out, crafted_out, bcast_rows, bcast_ld, batch,
                                batch_stride, d, bcast_batch_stride, stream, each);
}

// Attack-success metrics of a batch (afl_attack_metrics_batched; fs != NULL: afl_attack_metrics_batched_each).
// Workspace: [ProblemParams table][partial sums: double2[batch][tiles]]; the scalar call leaves the table unused.
static size_t metrics_partial_bytes(int batch, int64_t d, int dtype) {
  return align_up(static_cast<size_t>(batch) * colstats::deviation_tiles(d, dtype) * sizeof(double2), 256);
}

// rows != NULL (afl_attack_metrics_batched_rows, fs required): problem b has rows[b] rows, in [1, n].
static int attack_metrics(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, int f,
                          const int* fs, const float* agg, const int* idx, const int* sel, int sel_ld, float* dev_out,
                          double* sums_out, float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* ws,
                          size_t ws_bytes, cudaStream_t stream, const int* rows = nullptr) {
  const char* who = rows ? "afl_attack_metrics_batched_rows" : fs ? "afl_attack_metrics_batched_each" : "afl_attack_metrics_batched";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc) return rc;
  int fmin = f, fmax = f;
  if (fs && (rc = check_counts(who, fs, batch, INT32_MAX, &fmin, &fmax))) return rc;
  for (int b = 0; rows && b < batch; ++b)
    if (rows[b] < 1 || rows[b] > n) {
      set_error("%s: row count %d of problem %d is outside [1, %d]", who, rows[b], b, n);
      return AFL_ERR_BAD_ARG;
    }
  if (fmin < 0) { set_error("%s: corrupted_count %d is negative", who, f); return AFL_ERR_BAD_ARG; }
  if (agg && idx) { set_error("%s: give the aggregate as agg or as idx, not both", who); return AFL_ERR_BAD_ARG; }
  if ((dev_out || sums_out) && !agg && !idx) {
    set_error("%s: dev_out and sums_out need an aggregate (agg or idx)", who);
    return AFL_ERR_BAD_ARG;
  }
  if (krum_hit && !idx) { set_error("%s: krum_hit needs idx", who); return AFL_ERR_BAD_ARG; }
  if ((mal_count || sel_count) && !sel) { set_error("%s: mal_count and sel_count need sel", who); return AFL_ERR_BAD_ARG; }
  if (sel && sel_ld < 1) { set_error("%s: sel_ld must be >= 1 (got %d)", who, sel_ld); return AFL_ERR_BAD_ARG; }
  const bool pass = dev_out || sums_out || honest_out;          // the column pass and its partial sums
  const size_t need = table_bytes(batch) + metrics_partial_bytes(batch, d, dtype);
  if ((fs || pass) && (!ws || ws_bytes < need || reinterpret_cast<uintptr_t>(ws) % 256 != 0)) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  const ProblemParams* each = nullptr;
  if (fs) {
    rc = upload_table(who, batch, ws, ws_bytes, need, stream, [&](int b, ProblemParams& q) {
      q.f = fs[b];
      if (rows) q.tm.n_rows = rows[b];
    }, &each);
    if (rc) return rc;
  }
  return colstats::attack_metrics(G, batch, batch_stride, n, d, ld, dtype, f, each, agg, idx, sel, sel_ld, dev_out,
                                  sums_out, honest_out, krum_hit, mal_count, sel_count,
                                  static_cast<uint8_t*>(ws) + table_bytes(batch), stream, rows != nullptr);
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
                          size_t ws_bytes, cudaStream_t stream, const ProblemParams** each) {
  return upload_table(who, batch, ws, ws_bytes, table_bytes(batch), stream, [&](int b, ProblemParams& q) {
    q.f = fs[b];
    q.z = static_cast<float>(zs[b]);
    q.lr = static_cast<float>(lrs[b]);
    q.write = fs[b] > 0 && zs[b] != 0.0;               // malicious.py:20-21: z == 0 computes the statistics only
  }, each);
}

static int backdoor_start(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                          const int* fs, const double* zs, const double* lrs, const float* w, int64_t w_batch_stride,
                          float* mu_out, float* sigma_out, float* initial_out, void* ws, size_t ws_bytes,
                          cudaStream_t stream) {
  const char* who = "afl_backdoor_start_batched";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc) return rc;
  if (!w || !mu_out || !sigma_out || !initial_out) { set_error("%s: w and every output are required", who); return AFL_ERR_BAD_ARG; }
  if (w_batch_stride < 0 || (w_batch_stride > 0 && w_batch_stride < d)) {
    set_error("%s: w_batch_stride %lld must be 0 (one shared w) or >= d", who, static_cast<long long>(w_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  int fmax = 0;
  if ((rc = backdoor_values(who, batch, fs, n, zs, lrs, &fmax))) return rc;
  const ProblemParams* each = nullptr;
  if ((rc = backdoor_table(who, batch, fs, zs, lrs, ws, ws_bytes, stream, &each))) return rc;
  return colstats::backdoor_start(G, fmax, d, ld, dtype, batch, batch_stride, each, w, w_batch_stride, mu_out,
                                  sigma_out, initial_out, stream);
}

static int backdoor_finish(int batch, int64_t d, const int* fs, const double* zs, const double* lrs, const float* mu,
                           const float* sigma, const float* initial, const float* mal, int64_t mal_batch_stride,
                           float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* ws,
                           size_t ws_bytes, cudaStream_t stream) {
  const char* who = "afl_backdoor_finish_batched";
  if (!mu || !sigma || !initial || !mal || !crafted_out || d < 1) { set_error("%s: bad argument", who); return AFL_ERR_BAD_ARG; }
  if (batch < 1) { set_error("%s: batch must be >= 1 (got %d)", who, batch); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (batch > 1 && mal_batch_stride < d) {
    set_error("%s: mal_batch_stride %lld makes problems overlap", who, static_cast<long long>(mal_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  int fmax = 0;
  int rc = backdoor_values(who, batch, fs, INT32_MAX, zs, lrs, &fmax);
  if (rc) return rc;
  if (bcast_rows && fmax > 0 &&
      (bcast_ld < d || (batch > 1 && bcast_batch_stride < static_cast<int64_t>(fmax - 1) * bcast_ld + d))) {
    set_error("%s: bcast_ld / bcast_batch_stride make the written rows overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  const ProblemParams* each = nullptr;
  if ((rc = backdoor_table(who, batch, fs, zs, lrs, ws, ws_bytes, stream, &each))) return rc;
  return colstats::backdoor_finish(batch, d, each, mu, sigma, initial, mal, mal_batch_stride, crafted_out, bcast_rows,
                                   bcast_batch_stride, bcast_ld, stream);
}

// ------------------------------------------------------------------------------------------------
// Device-parameter calls (afl_*_dev): the per-problem arrays are device memory, so a call never reads them on the host.
// problem_table_kernel builds the table the host calls above build, one thread per problem, and runs their per-problem
// checks in the same order.  A problem that fails a check gets its first code in the caller's sticky status[b] and
// the safe row of rows_b = n, users_count_b = n, f_b = 0, which keeps every kernel inside its slot; its outputs are
// then not the reference's, and only status says so.  After the host checks of shapes, pointers and the workspace,
// a call makes no host copy, synchronisation or allocation, so it can be captured into a CUDA graph.
// ------------------------------------------------------------------------------------------------
enum TableRule { T_ALIE = B_BULYAN + 1, T_METRICS };

struct TableArgs {
  int rule;                   // BatchedRule, T_ALIE or T_METRICS
  int batch, n;
  const int* rows;            // NULL: n rows in every problem
  const int* ucs;             // NULL: users_count without rows, rows with them
  int users_count;
  const int* fs;
  const double* zs;           // ALIE only
  ProblemParams* table;
  int* status;
  const int* sel;             // Bulyan's second stage: rows of sel_ld entries, sel[b][theta_b - 1] < 0 = failed round
  int sel_ld;
};

// The first code of the host calls' checks for one problem: afl_defend_batched_rows / _each (rows = n),
// afl_alie_batched_each, afl_attack_metrics_batched_rows / _each.
__device__ int problem_code(int rule, int n, bool ragged, int m, int uc, int f) {
  if (rule == T_ALIE) return f < 0 || f > n ? AFL_ERR_BAD_ARG : AFL_OK;
  if (f < 0 || (rule != T_METRICS && f > INT32_MAX / 4)) return AFL_ERR_BAD_ARG;
  if (ragged && (m < 1 || m > n)) return AFL_ERR_BAD_ARG;
  if (rule == B_KRUM && uc < 2 * static_cast<int64_t>(f) + 1) return AFL_ERR_PRECONDITION;
  if (rule == B_BULYAN && uc < 4 * static_cast<int64_t>(f) + 3) return AFL_ERR_PRECONDITION;
  if (rule == B_BULYAN && uc != m) return AFL_ERR_UNSUPPORTED;
  return AFL_OK;
}

__global__ void __launch_bounds__(128) problem_table_kernel(const TableArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.batch) return;
  int f = a.fs[b];
  int m = a.rows ? a.rows[b] : a.n;
  int uc = a.ucs ? a.ucs[b] : a.rows ? m : a.users_count;
  const int code = problem_code(a.rule, a.n, a.rows != nullptr, m, uc, f);
  if (code != AFL_OK) { m = a.n; uc = a.n; f = 0; }
  ProblemParams q{};
  q.f = f;
  if (a.rule == T_ALIE) {
    q.z = static_cast<float>(a.zs[b]);
    q.write = f > 0 && a.zs[b] != 0.0;                  // malicious.py:20-21: z == 0 computes the statistics only
  } else if (a.rule == T_METRICS) {
    if (a.rows) q.tm.n_rows = m;
  } else {
    q.take = select::krum_take(m, uc, f);
    q.theta = uc - 2 * f;
    // Bulyan's second stage: the trimmed mean of the theta_b selected rows with 2 f_b (the whole-slot call's only table)
    q.tm = a.rule == B_BULYAN && (a.sel || !a.rows) ? tmean::shape(q.theta, 2 * f) : tmean::shape(m, f);
  }
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
// them class by class and in problem order within a class (upload_class_table's order), and start[kSlotClasses + 1]
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
  if (!ws || ws_bytes < need || reinterpret_cast<uintptr_t>(ws) % 256 != 0) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, ws_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  return AFL_OK;
}

static int table_dev(const char* rule, int batch, int n, const int* rows, int users_count, const int* ucs,
                     const int* fs, const double* zs, void* ws, size_t ws_bytes, int* status, cudaStream_t stream) {
  const char* who = "afl_batched_table_dev";
  const bool alie = rule && !strcmp(rule, "ALIE"), metrics = rule && !strcmp(rule, "AttackMetrics");
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD && !alie && !metrics) { set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)"); return AFL_ERR_BAD_ARG; }
  if (batch < 1 || n < 1) { set_error("%s: batch and n must be >= 1 (got %d, %d)", who, batch, n); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (alie && !zs) { set_error("%s: the per-problem attack strengths are NULL", who); return AFL_ERR_BAD_ARG; }
  int rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch));
  if (rc) return rc;
  TableArgs a{};
  a.rule = alie ? static_cast<int>(T_ALIE) : metrics ? static_cast<int>(T_METRICS) : static_cast<int>(r);
  a.batch = batch; a.n = n; a.rows = alie ? nullptr : rows; a.ucs = rows ? ucs : nullptr; a.users_count = users_count;
  a.fs = fs; a.zs = zs; a.table = static_cast<ProblemParams*>(ws); a.status = status;
  return launch_table(a, stream);
}

// afl_defend_batched_rows (rows != NULL) or afl_defend_batched_each (rows == NULL, n rows and users_count in every
// problem) with device arrays: the same kernels on a device-built table.  Host scalars of those calls become bounds
// that hold for every accepted value: Bulyan's selection width is the caller's sel_ld >= n >= theta_b (the host calls
// use theta_max), and the corrupted counts and users counts that only fill fields a table overrides are passed as 0.
static int defend_batched_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                              int64_t ld, int dtype, const int* rows, int users_count, const int* ucs, const int* fs,
                              float* out, int* idx_out, int* sel_out, int sel_ld, void* ws, size_t ws_bytes,
                              int* status, cudaStream_t stream) {
  const char* who = "afl_defend_batched_dev";
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD) { set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)"); return AFL_ERR_BAD_ARG; }
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype);
  if (rc) return rc;
  if ((r != B_KRUM && !out) || (r == B_KRUM && !idx_out) || (r == B_BULYAN && !sel_out)) {
    set_error("%s: %s needs %s", who, rule, r == B_KRUM ? "idx_out" : r == B_BULYAN ? "out and sel_out" : "out");
    return AFL_ERR_BAD_ARG;
  }
  if (r == B_BULYAN && sel_ld < n) {
    set_error("%s: Bulyan's selection width sel_ld (%d) must be at least n (%d)", who, sel_ld, n);
    return AFL_ERR_BAD_ARG;
  }
  size_t gram_ws = 0, tabs = 0;
  const size_t rule_ws = batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch) + rule_ws))) return rc;

  TableArgs a{};
  a.rule = r; a.batch = batch; a.n = n; a.rows = rows; a.ucs = rows ? ucs : nullptr; a.users_count = users_count;
  a.fs = fs; a.table = static_cast<ProblemParams*>(ws); a.status = status;
  if ((rc = launch_table(a, stream))) return rc;
  const ProblemParams* each = a.table;
  const ProblemParams* ragged = rows ? each : nullptr;
  if (r == B_MEAN) return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream, ragged);
  if (r == B_TM) return tmean::trimmed_mean_batched(G, n, d, ld, dtype, nullptr, n, 0, out, batch, batch_stride, 0, d, stream, each);
  uint8_t* p = static_cast<uint8_t*>(ws) + table_bytes(batch);
  const size_t nn = static_cast<size_t>(batch) * n * n;
  double* d2 = reinterpret_cast<double*>(p);
  float* dist = reinterpret_cast<float*>(p + align_up(nn * 8, 256));
  void* sel_ws = p + tabs + gram_ws;
  const size_t sel_ws_bytes = ws_bytes - table_bytes(batch) - tabs - gram_ws;
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, d2, p + tabs, gram_ws, 0, stream, ragged);
  if (rc) return rc;
  if (r == B_KRUM) return select::krum_from_sqdist(d2, n, 0, 0, idx_out, sel_ws, sel_ws_bytes, stream, batch, each, rows != nullptr);
  rc = gram::sqdist_to_dist(d2, n, dist, stream, batch); if (rc) return rc;
  rc = select::bulyan_rounds(dist, n, 0, sel_ld, sel_out, sel_ws, sel_ws_bytes, stream, batch, each, rows != nullptr);
  if (rc) return rc;
  a.sel = sel_out; a.sel_ld = sel_ld;                    // second stage's table, and a failed round's status
  if ((rc = launch_table(a, stream))) return rc;
  return tmean::trimmed_mean_batched(G, n, d, ld, dtype, sel_out, n, 0, out, batch, batch_stride, sel_ld, d, stream, each);
}

// afl_defend_batched_large with device arrays (afl_defend_batched_large_dev): n <= 128 is afl_defend_batched_dev.  Above,
// the workspace is the large call's (ProblemParams[batch], perm[batch], then the rule's scratch) followed by one
// kClassStartBytes block for start[].  After each table launch class_perm_kernel groups the problems on the device, and
// the trimmed mean runs one device-count launch per class (tmean::trimmed_mean_classes_dev).  Every kernel reads the
// table as afl_defend_batched_large does, except the Gram without rows: with n rows in every problem its multi-tile
// centre is the same without the table, and the table of a whole-slot Bulyan holds the second stage's tm already.
static int defend_batched_large_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                                    int64_t ld, int dtype, const int* rows, int users_count, const int* ucs,
                                    const int* fs, float* out, int* idx_out, int* sel_out, int sel_ld, void* ws,
                                    size_t ws_bytes, int* status, cudaStream_t stream) {
  const char* who = "afl_defend_batched_large_dev";
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD) { set_error("%s: unknown rule '%s'", who, rule ? rule : "(null)"); return AFL_ERR_BAD_ARG; }
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, kBatchLargeMaxClients);
  if (rc) return rc;
  if (n <= kBatchMaxClients)
    return defend_batched_dev(rule, G, batch, batch_stride, n, d, ld, dtype, rows, users_count, ucs, fs, out, idx_out,
                              sel_out, sel_ld, ws, ws_bytes, status, stream);
  if ((r != B_KRUM && !out) || (r == B_KRUM && !idx_out) || (r == B_BULYAN && !sel_out)) {
    set_error("%s: %s needs %s", who, rule, r == B_KRUM ? "idx_out" : r == B_BULYAN ? "out and sel_out" : "out");
    return AFL_ERR_BAD_ARG;
  }
  if (r == B_BULYAN && sel_ld < n) {
    set_error("%s: Bulyan's selection width sel_ld (%d) must be at least n (%d)", who, sel_ld, n);
    return AFL_ERR_BAD_ARG;
  }
  size_t gram_ws = 0, tabs = 0;
  const size_t rule_ws = batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
  const size_t tab_bytes = class_table_bytes(batch, n);
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, tab_bytes + rule_ws + kClassStartBytes))) return rc;

  TableArgs a{};
  a.rule = r; a.batch = batch; a.n = n; a.rows = rows; a.ucs = rows ? ucs : nullptr; a.users_count = users_count;
  a.fs = fs; a.table = static_cast<ProblemParams*>(ws); a.status = status;
  const ProblemParams* each = a.table;
  uint8_t* p = static_cast<uint8_t*>(ws) + tab_bytes;
  int* perm = reinterpret_cast<int*>(static_cast<uint8_t*>(ws) + static_cast<size_t>(batch) * sizeof(ProblemParams));
  int* start = reinterpret_cast<int*>(p + rule_ws);
  if ((rc = launch_table(a, stream))) return rc;
  if (r == B_MEAN) return colstats::mean_batched(G, n, d, ld, dtype, out, batch, batch_stride, d, stream, each);
  if (r == B_TM) {
    if ((rc = launch_class_perm(each, batch, perm, start, stream))) return rc;
    return tmean::trimmed_mean_classes_dev(G, n, d, ld, dtype, nullptr, out, batch, batch_stride, 0, d, stream, each,
                                           perm, start);
  }
  const size_t nn = static_cast<size_t>(batch) * n * n;
  double* d2 = reinterpret_cast<double*>(p);
  float* dist = reinterpret_cast<float*>(p + align_up(nn * 8, 256));
  void* sel_ws = p + tabs + gram_ws;
  const size_t sel_ws_bytes = rule_ws - tabs - gram_ws;
  rc = gram::sqdist_batched(G, batch, batch_stride, n, d, ld, dtype, d2, p + tabs, gram_ws, 0, stream,
                            rows ? each : nullptr);
  if (rc) return rc;
  if (r == B_KRUM) return select::krum_from_sqdist(d2, n, 0, 0, idx_out, sel_ws, sel_ws_bytes, stream, batch, each, true);
  rc = gram::sqdist_to_dist(d2, n, dist, stream, batch); if (rc) return rc;
  rc = select::bulyan_rounds(dist, n, 0, sel_ld, sel_out, sel_ws, sel_ws_bytes, stream, batch, each, true);
  if (rc) return rc;
  a.sel = sel_out; a.sel_ld = sel_ld;                    // second stage's table (theta_b classes), and a failed round's status
  if ((rc = launch_table(a, stream))) return rc;
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
  if (bcast_rows && (bcast_ld < d || (batch > 1 && bcast_batch_stride < static_cast<int64_t>(n - 1) * bcast_ld + d))) {
    set_error("%s: bcast_ld / bcast_batch_stride make the written rows overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch)))) return rc;
  TableArgs a{};
  a.rule = T_ALIE; a.batch = batch; a.n = n; a.fs = fs; a.zs = zs; a.table = static_cast<ProblemParams*>(ws); a.status = status;
  if ((rc = launch_table(a, stream))) return rc;
  return colstats::alie_batched_dev(G, n, d, ld, dtype, mu_out, sigma_out, crafted_out, bcast_rows, bcast_ld, batch,
                                    batch_stride, d, bcast_batch_stride, stream, a.table);
}

// The backdoor crafting's table from device arrays (afl_backdoor_start_batched_dev / _finish_batched_dev): backdoor_table's
// row, with the host calls' count check per problem (f_b < 0 or f_b > n -> AFL_ERR_BAD_ARG, and the safe f_b = 0).
__global__ void __launch_bounds__(128) backdoor_table_kernel(int batch, int n, const int* fs, const double* zs,
                                                             const double* lrs, ProblemParams* table, int* status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  int f = fs[b];
  const int code = f < 0 || f > n ? AFL_ERR_BAD_ARG : AFL_OK;
  if (code != AFL_OK) f = 0;
  ProblemParams q{};
  q.f = f;
  q.z = static_cast<float>(zs[b]);
  q.lr = static_cast<float>(lrs[b]);
  q.write = f > 0 && zs[b] != 0.0;                      // malicious.py:20-21: z == 0 computes the statistics only
  table[b] = q;
  if (code != AFL_OK && status[b] == AFL_OK) status[b] = code;
}

static int backdoor_table_dev(const char* who, int batch, int n, const int* fs, const double* zs, const double* lrs,
                              void* ws, size_t ws_bytes, int* status, cudaStream_t stream) {
  if (!zs || !lrs) { set_error("%s: the per-problem attack strengths or learning rates are NULL", who); return AFL_ERR_BAD_ARG; }
  int rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch));
  if (rc) return rc;
  backdoor_table_kernel<<<static_cast<unsigned>((batch + 127) / 128), 128, 0, stream>>>(
      batch, n, fs, zs, lrs, static_cast<ProblemParams*>(ws), status);
  AFL_LAUNCH_CHECK("backdoor_table_kernel");
  return AFL_OK;
}

// afl_backdoor_start_batched with device arrays: n bounds every f_b (the host call's fmax).
static int backdoor_start_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                              const int* fs, const double* zs, const double* lrs, const float* w, int64_t w_batch_stride,
                              float* mu_out, float* sigma_out, float* initial_out, void* ws, size_t ws_bytes,
                              int* status, cudaStream_t stream) {
  const char* who = "afl_backdoor_start_batched_dev";
  int rc = check_batch(who, G, batch, batch_stride, n, d, ld, dtype, INT32_MAX);
  if (rc) return rc;
  if (!w || !mu_out || !sigma_out || !initial_out) { set_error("%s: w and every output are required", who); return AFL_ERR_BAD_ARG; }
  if (w_batch_stride < 0 || (w_batch_stride > 0 && w_batch_stride < d)) {
    set_error("%s: w_batch_stride %lld must be 0 (one shared w) or >= d", who, static_cast<long long>(w_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
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
  if (batch < 1) { set_error("%s: batch must be >= 1 (got %d)", who, batch); return AFL_ERR_BAD_ARG; }
  if (batch > kBatchMax) { set_error("%s: batch <= %d problems (got %d)", who, kBatchMax, batch); return AFL_ERR_UNSUPPORTED; }
  if (batch > 1 && mal_batch_stride < d) {
    set_error("%s: mal_batch_stride %lld makes problems overlap", who, static_cast<long long>(mal_batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  if (bcast_rows && (bcast_ld < d || (batch > 1 && bcast_batch_stride < static_cast<int64_t>(n - 1) * bcast_ld + d))) {
    set_error("%s: bcast_ld / bcast_batch_stride make the written rows overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  int rc = backdoor_table_dev(who, batch, n, fs, zs, lrs, ws, ws_bytes, status, stream);
  if (rc) return rc;
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
  if (rc) return rc;
  if (agg && idx) { set_error("%s: give the aggregate as agg or as idx, not both", who); return AFL_ERR_BAD_ARG; }
  if ((dev_out || sums_out) && !agg && !idx) {
    set_error("%s: dev_out and sums_out need an aggregate (agg or idx)", who);
    return AFL_ERR_BAD_ARG;
  }
  if (krum_hit && !idx) { set_error("%s: krum_hit needs idx", who); return AFL_ERR_BAD_ARG; }
  if ((mal_count || sel_count) && !sel) { set_error("%s: mal_count and sel_count need sel", who); return AFL_ERR_BAD_ARG; }
  if (sel && sel_ld < 1) { set_error("%s: sel_ld must be >= 1 (got %d)", who, sel_ld); return AFL_ERR_BAD_ARG; }
  if ((rc = check_dev(who, fs, status, ws, ws_bytes, table_bytes(batch) + metrics_partial_bytes(batch, d, dtype)))) return rc;
  TableArgs a{};
  a.rule = T_METRICS; a.batch = batch; a.n = n; a.rows = rows; a.fs = fs; a.table = static_cast<ProblemParams*>(ws);
  a.status = status;
  if ((rc = launch_table(a, stream))) return rc;
  return colstats::attack_metrics(G, batch, batch_stride, n, d, ld, dtype, 0, a.table, agg, idx, sel, sel_ld, dev_out,
                                  sums_out, honest_out, krum_hit, mal_count, sel_count,
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
  size_t gram_ws = 0, tabs = 0;
  return batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
}

size_t afl_batched_each_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const bool alie = rule && !strcmp(rule, "ALIE");
  const BatchedRule r = batched_rule(rule);
  if ((r == B_BAD && !alie) || batch < 1 || batch > kBatchMax || n < 1 || n > kBatchMaxClients || d < 1) return 0;
  size_t gram_ws = 0, tabs = 0;
  return table_bytes(batch) + batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
}

int afl_defend_batched(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                       int dtype, int users_count, int corrupted_count, float* out, int* idx_out, int* sel_out,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return defend_batched(rule, G, batch, batch_stride, n, d, ld, dtype, users_count, corrupted_count, nullptr, out, idx_out,
                        sel_out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int afl_defend_batched_each(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                            int64_t ld, int dtype, int users_count, const int* corrupted_counts, float* out, int* idx_out,
                            int* sel_out, void* workspace, size_t workspace_bytes, void* stream) {
  if (!corrupted_counts) {
    set_error("afl_defend_batched_each: the per-problem corrupted counts are NULL");
    return AFL_ERR_BAD_ARG;
  }
  return defend_batched(rule, G, batch, batch_stride, n, d, ld, dtype, users_count, 0, corrupted_counts, out, idx_out,
                        sel_out, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
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
  return defend_batched_rows("afl_defend_batched_rows", kBatchMaxClients, rule, G, batch, batch_stride, n, d, ld, dtype,
                             rows, users_counts, corrupted_counts, out, idx_out, sel_out, workspace, workspace_bytes,
                             static_cast<cudaStream_t>(stream));
}

size_t afl_batched_large_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype) {
  const BatchedRule r = batched_rule(rule);
  if (r == B_BAD || n < 1 || n > kBatchLargeMaxClients) return 0;
  if (n <= kBatchMaxClients) return afl_batched_rows_workspace_bytes(rule, batch, n, d, dtype);
  if (batch < 1 || batch > kBatchMax || d < 1 || (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16)) return 0;
  size_t gram_ws = 0, tabs = 0;
  return class_table_bytes(batch, n) + batched_ws_parts(r, batch, n, d, dtype, &gram_ws, &tabs);
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
  return defend_batched_rows("afl_defend_batched_large", kBatchLargeMaxClients, rule, G, batch, batch_stride, n, d, ld,
                             dtype, rows, users_counts, corrupted_counts, out, idx_out, sel_out, workspace,
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
  return defend_batched_dev(rule, G, batch, batch_stride, n, d, ld, dtype, rows, users_count, users_counts,
                            corrupted_counts, out, idx_out, sel_out, sel_ld, workspace, workspace_bytes, status,
                            static_cast<cudaStream_t>(stream));
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
  return defend_batched_large_dev(rule, G, batch, batch_stride, n, d, ld, dtype, rows, users_count, users_counts,
                                  corrupted_counts, out, idx_out, sel_out, sel_ld, workspace, workspace_bytes, status,
                                  static_cast<cudaStream_t>(stream));
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
