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
int sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out, void* ws, size_t ws_bytes,
                   int flags, cudaStream_t stream);
int sqdist_to_dist(const double* d2, int n, float* dist, cudaStream_t stream);
}
namespace select {
int max_clients();
size_t workspace_bytes(int n);
int krum_select(const float* dist, int n, int users_count, int corrupted_count, int* idx_out, float* scores_out,
                void* ws, size_t ws_bytes, cudaStream_t stream);
int krum_from_sqdist(const double* d2, int n, int users_count, int corrupted_count, int* idx_out, void* ws,
                     size_t ws_bytes, cudaStream_t stream);
int bulyan_select(const float* dist, int n, int users_count, int f, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream);
}
namespace tmean {
int trimmed_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                 int corrupted_count, float* out, cudaStream_t stream);
}
namespace colstats {
int mean(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, cudaStream_t stream);
int alie(const void* G, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
         float* crafted_out, float* bcast, int64_t bcast_ld, cudaStream_t stream);
int gather_row(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* idx_dev, float* out,
               cudaStream_t stream);
int momentum_step(float* w, float* v, const float* g, int64_t d, float momentum, float lr, cudaStream_t stream);
int alie_band(const float* mu, const float* sigma, double z, const float* x, float* out, int64_t d, cudaStream_t stream);
}

__global__ void add_f64_kernel(double* __restrict__ acc, const double* __restrict__ x, size_t n, int first) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) acc[i] = first ? x[i] : acc[i] + x[i];
}

// ------------------------------------------------------------------------------------------------
// Host-buffer path: the matrix stays in host memory and is streamed through a bounded device staging area.
//
//   * Column slabs of `slab_cols` columns go through a ring of kRingSlots device slots: the copy stream fills
//     slot s % slots while the compute stream runs the kernels of the slab before it.  `freed[slot]` is
//     recorded on the compute stream after the last kernel that reads the slot, and the copy stream waits on
//     it before overwriting the slot.
//   * Krum sums one d2 table per slab (sqdist_partial + add_f64_kernel, in slab order); TrimmedMean and
//     NoDefense finish each slab's columns as soon as its kernel has run.
//   * Bulyan keeps slabs 0 .. R-1 resident (as many as the budget holds) and streams the rest.  After
//     selection, stage 2 runs once over the resident columns with row_index = sel; for the other columns it
//     re-streams only the theta selected rows, packed in selection order, and runs the same trimmed mean with
//     row_index = NULL.  When the whole matrix fits, R covers every slab and nothing is streamed twice.
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
  void* small = nullptr; size_t small_bytes = 0;    // d2 tables, dist, indices, output vector
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

static int defend_host(const char* rule, const float* G, int n, int64_t d, int64_t ld, int users_count, int f,
                       float* out_host, int* idx_out, int64_t slab_cols) {
  enum { R_MEAN, R_KRUM, R_TM, R_BULYAN } r;
  if (!strcmp(rule, "NoDefense")) r = R_MEAN;
  else if (!strcmp(rule, "Krum")) r = R_KRUM;
  else if (!strcmp(rule, "TrimmedMean")) r = R_TM;
  else if (!strcmp(rule, "Bulyan")) r = R_BULYAN;
  else { set_error("afl_defend_host: unknown rule '%s'", rule); return AFL_ERR_BAD_ARG; }
  if (!G || n < 1 || d < 1 || ld < d) { set_error("afl_defend_host: bad argument"); return AFL_ERR_BAD_ARG; }
  if (r != R_KRUM && !out_host) { set_error("afl_defend_host: out_host is required for %s", rule); return AFL_ERR_BAD_ARG; }
  // the reference's asserts (defences.py:24-25, :56)
  if (r == R_KRUM && users_count < 2 * f + 1) {
    set_error("krum: users_count >= 2*corrupted_count + 1 violated (%d, %d)", users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if (r == R_BULYAN && users_count < 4 * f + 3) {
    set_error("bulyan: users_count >= 4*corrupted_count + 3 violated (%d, %d)", users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if ((r == R_KRUM || r == R_BULYAN) && n > select::max_clients()) {   // before any copy or launch
    set_error("afl_defend_host: %s supports n <= %d clients (got %d)", rule, select::max_clients(), n);
    return AFL_ERR_UNSUPPORTED;
  }
  HostCtx& c = g_ctx[current_device()];          // streams, events and buffers belong to the current device
  std::lock_guard<std::mutex> lock(c.mu);
  if (!c.init) {
    AFL_CUDA(cudaStreamCreateWithFlags(&c.copy, cudaStreamNonBlocking));
    AFL_CUDA(cudaStreamCreateWithFlags(&c.comp, cudaStreamNonBlocking));
    AFL_CUDA(cudaEventCreateWithFlags(&c.ready, cudaEventDisableTiming));
    for (auto& e : c.freed) AFL_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c.init = true;
  }
  struct Drain {                                  // every return leaves both streams idle: no copy still reads G
    HostCtx& c;
    ~Drain() { cudaStreamSynchronize(c.copy); cudaStreamSynchronize(c.comp); }
  } drain{c};
  const bool table = r == R_KRUM || r == R_BULYAN;
  const int theta = r == R_BULYAN ? users_count - 2 * f : 0;
  const int64_t ld_dev = (d + 31) / 32 * 32;          // padded pitch: TMA + 16-byte loads always apply
  if (slab_cols <= 0) slab_cols = (int64_t(96) << 20) / (static_cast<int64_t>(n) * 4);   // ~96 MB per slab
  slab_cols = (slab_cols + 31) / 32 * 32;
  if (slab_cols < 32) slab_cols = 32;
  if (slab_cols > ld_dev) slab_cols = ld_dev;         // one slab either way; keeps the slots no wider than the matrix
  const int nslab = static_cast<int>((d + slab_cols - 1) / slab_cols);
  const size_t nn = static_cast<size_t>(n) * n;
  const int sel_len = n > theta ? n : theta;         // also the rows of a slot: Bulyan's second pass packs theta rows

  // ---- device footprint: workspaces and tables (fixed), then the resident prefix and the ring
  const size_t gram_ws_bytes = table ? align_up(gram::workspace_bytes(n, slab_cols, AFL_F32, 0), 256) : 0;
  const size_t ws_need = table ? gram_ws_bytes + select::workspace_bytes(n) : 256;
  const size_t small_need = (table ? align_up(nn * 8, 256) * 2 + align_up(nn * 4, 256) : 0) +
                            align_up(static_cast<size_t>(sel_len) * 4, 256) +
                            (r != R_KRUM ? align_up(static_cast<size_t>(d) * 4, 256) : 0) + 1024;
  const size_t slab_bytes = static_cast<size_t>(n) * slab_cols * sizeof(float);
  const size_t slot_bytes = align_up(static_cast<size_t>(sel_len) * slab_cols * sizeof(float), 256);
  size_t free_b = 0, total_b = 0;
  AFL_CUDA(cudaMemGetInfo(&free_b, &total_b));
  const size_t budget = host_budget(free_b, c.stage_bytes + c.ws_bytes + c.small_bytes);
  const size_t fixed = ws_need + small_need;
  const size_t full_res = align_up(static_cast<size_t>(n) * ld_dev * sizeof(float), 256);
  int R = 0, slots = 0;                               // resident slabs, ring slots
  if (r == R_BULYAN && fixed + full_res <= budget) {
    R = nslab;
  } else {
    const int min_slots = nslab < 2 ? nslab : 2;
    if (fixed + min_slots * slot_bytes > budget) {
      set_error("afl_defend_host: needs %zu bytes of device memory (%d staging slots of %zu bytes for %lld-column slabs, "
                "plus %zu bytes of tables and workspaces) but may use %zu (free memory less 1 GiB, capped by "
                "AFL_HOST_DEVICE_BYTES); use narrower slabs or a larger budget",
                fixed + min_slots * slot_bytes, min_slots, slot_bytes, static_cast<long long>(slab_cols), fixed, budget);
      return AFL_ERR_UNSUPPORTED;
    }
    slots = min_slots;
    if (r == R_BULYAN) {                              // spend the rest on resident slabs: they are not re-streamed
      const size_t spare = budget - fixed - slots * slot_bytes;
      const size_t fit = spare > 256 ? (spare - 256) / slab_bytes : 0;
      R = static_cast<int>(fit < static_cast<size_t>(nslab - 1) ? fit : static_cast<size_t>(nslab - 1));
    } else {
      const int most = nslab < kRingSlots ? nslab : kRingSlots;
      while (slots < most && fixed + (slots + 1) * slot_bytes <= budget) ++slots;
    }
  }
  const int64_t ld_res = R == nslab ? ld_dev : R * slab_cols;   // resident pitch
  const int64_t d_res = R == nslab ? d : R * slab_cols;        // resident columns
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

  uint8_t* sp = static_cast<uint8_t*>(c.small);
  double* d2_acc = nullptr; double* d2_part = nullptr; float* dist = nullptr;
  if (table) {
    d2_acc = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256);
    d2_part = reinterpret_cast<double*>(sp); sp += align_up(nn * 8, 256);
    dist = reinterpret_cast<float*>(sp); sp += align_up(nn * 4, 256);
  }
  int* sel = reinterpret_cast<int*>(sp); sp += align_up(static_cast<size_t>(sel_len) * 4, 256);
  float* out_dev = reinterpret_cast<float*>(sp);
  float* res = static_cast<float*>(c.stage);
  float* ring = reinterpret_cast<float*>(static_cast<uint8_t*>(c.stage) + res_bytes);
  const int64_t slot_elems = static_cast<int64_t>(slot_bytes / sizeof(float));
  void* gram_ws = c.ws;
  void* sel_ws = static_cast<uint8_t*>(c.ws) + gram_ws_bytes;
  const size_t sel_ws_bytes = c.ws_bytes - gram_ws_bytes;
  int rc = AFL_OK;
  int64_t ring_i = 0;                                 // ring slabs issued so far (pass 1 and pass 2)

  // next ring slot: the copy stream waits until the compute stream has finished reading it
  auto next_slot = [&](int* slot, float** m) -> cudaError_t {
    *slot = static_cast<int>(ring_i % slots);
    *m = ring + *slot * slot_elems;
    return ring_i++ >= slots ? cudaStreamWaitEvent(c.copy, c.freed[*slot], 0) : cudaSuccess;
  };

  // ---- pass 1: every column once
  for (int s = 0; s < nslab; ++s) {
    const int64_t c0 = static_cast<int64_t>(s) * slab_cols;
    const int64_t w = (d - c0 < slab_cols) ? d - c0 : slab_cols;
    int slot = -1;
    float* m = res + c0;
    if (s >= R) AFL_CUDA(next_slot(&slot, &m));
    const int64_t mld = s < R ? ld_res : slab_cols;
    AFL_CUDA(cudaMemcpy2DAsync(m, mld * sizeof(float), G + c0, ld * sizeof(float), w * sizeof(float), n,
                               cudaMemcpyHostToDevice, c.copy));
    AFL_CUDA(cudaEventRecord(c.ready, c.copy));
    AFL_CUDA(cudaStreamWaitEvent(c.comp, c.ready, 0));
    if (table) {
      rc = gram::sqdist_partial(m, n, w, mld, AFL_F32, d2_part, gram_ws, gram_ws_bytes, 0, c.comp);
      if (rc) return rc;
      add_f64_kernel<<<static_cast<unsigned>((nn + 255) / 256), 256, 0, c.comp>>>(d2_acc, d2_part, nn, s == 0);
      AFL_LAUNCH_CHECK("add_f64_kernel");
    } else if (r == R_TM) {
      rc = tmean::trimmed_mean(m, n, w, mld, AFL_F32, nullptr, n, f, out_dev + c0, c.comp);
      if (rc) return rc;
    } else {
      rc = colstats::mean(m, n, w, mld, AFL_F32, out_dev + c0, c.comp);
      if (rc) return rc;
    }
    if (slot >= 0) AFL_CUDA(cudaEventRecord(c.freed[slot], c.comp));
  }
  if (r == R_KRUM) {
    int host_idx = -1;
    rc = select::krum_from_sqdist(d2_acc, n, users_count, f, sel, sel_ws, sel_ws_bytes, c.comp); if (rc) return rc;
    AFL_CUDA(cudaMemcpyAsync(&host_idx, sel, sizeof(int), cudaMemcpyDeviceToHost, c.comp));
    AFL_CUDA(cudaStreamSynchronize(c.comp));
    if (idx_out) *idx_out = host_idx;
    if (out_host) {                                   // the reference returns the winning ROW (a view)
      const int row = host_idx < 0 ? host_idx + n : host_idx;
      memcpy(out_host, G + static_cast<int64_t>(row) * ld, static_cast<size_t>(d) * sizeof(float));
    }
    return AFL_OK;
  }
  if (r == R_BULYAN) {
    rc = gram::sqdist_to_dist(d2_acc, n, dist, c.comp); if (rc) return rc;
    rc = select::bulyan_select(dist, n, users_count, f, sel, sel_ws, sel_ws_bytes, c.comp); if (rc) return rc;
    if (R > 0) {                                      // stage 2 over the resident columns
      rc = tmean::trimmed_mean(res, n, d_res, ld_res, AFL_F32, sel, theta, 2 * f, out_dev, c.comp); if (rc) return rc;
    }
    std::vector<int> hsel(static_cast<size_t>(theta));
    AFL_CUDA(cudaMemcpyAsync(hsel.data(), sel, static_cast<size_t>(theta) * sizeof(int), cudaMemcpyDeviceToHost, c.comp));
    AFL_CUDA(cudaStreamSynchronize(c.comp));
    if (hsel[theta - 1] < 0) {                        // a failed round marks itself and every later round with -1
      set_error("bulyan: a selection round found no eligible user (NaN or >= 1e20 scores); the reference raises KeyError(-1)");
      return AFL_ERR_NO_WINNER;
    }
    // ---- pass 2: the theta selected rows of the streamed columns, packed in selection order.  The kernel is
    // column-wise, so the slab may be as wide as a slot holds.
    const int64_t w2 = slot_elems / theta / 32 * 32;
    for (int64_t c0 = d_res; c0 < d; c0 += w2) {
      const int64_t w = (d - c0 < w2) ? d - c0 : w2;
      int slot = -1;
      float* m = nullptr;
      AFL_CUDA(next_slot(&slot, &m));
      for (int i = 0; i < theta; ++i) {
        const int row = hsel[i] < 0 ? hsel[i] + n : hsel[i];
        AFL_CUDA(cudaMemcpyAsync(m + static_cast<int64_t>(i) * w2, G + static_cast<int64_t>(row) * ld + c0,
                                 w * sizeof(float), cudaMemcpyHostToDevice, c.copy));
      }
      AFL_CUDA(cudaEventRecord(c.ready, c.copy));
      AFL_CUDA(cudaStreamWaitEvent(c.comp, c.ready, 0));
      rc = tmean::trimmed_mean(m, theta, w, w2, AFL_F32, nullptr, theta, 2 * f, out_dev + c0, c.comp); if (rc) return rc;
      AFL_CUDA(cudaEventRecord(c.freed[slot], c.comp));
    }
  }
  AFL_CUDA(cudaMemcpyAsync(out_host, out_dev, static_cast<size_t>(d) * sizeof(float), cudaMemcpyDeviceToHost, c.comp));
  AFL_CUDA(cudaStreamSynchronize(c.comp));
  if (idx_out) *idx_out = -1;
  return AFL_OK;
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

int afl_defend_host(const char* rule, const float* G_host, int n, int64_t d, int64_t ld, int users_count,
                    int corrupted_count, float* out_host, int* idx_out, int64_t slab_cols) {
  if (!rule) { set_error("afl_defend_host: rule is NULL"); return AFL_ERR_BAD_ARG; }
  return defend_host(rule, G_host, n, d, ld, users_count, corrupted_count, out_host, idx_out, slab_cols);
}

}  // extern "C"
