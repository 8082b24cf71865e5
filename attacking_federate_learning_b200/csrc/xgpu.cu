// The one exchange step of the D-sharded path (SURVEY 8e) over NVLink peer memory.
//
// Every rank owns ONE cudaMalloc'ed block, exported with cudaIpcGetMemHandle and mapped by its peers:
//     [table 0: n_max^2 float64][table 1][flags: world x u64][done counter]
// afl_sqdist_partial writes the rank's partial squared-distance table straight into table (epoch & 1); a one-thread
// `publish` kernel then stores the epoch into flags[rank] of EVERY rank (release, system scope).  A consumer kernel
// waits until all `world` flags of its own block have reached the epoch (acquire) and then reads the peers' tables
// through the mapped pointers, adding them in rank order -> the sum is bit-identical on every rank (selection stays
// replicated and deterministic, no broadcast), and there is no NCCL launch, no host round trip and no reduction
// tree on the latency path of an 80 KB (N = 100) .. 8 MB (N = 1000) table.  Two tables alternate by epoch: a rank can
// run at most one step ahead of the slowest peer (its consumer kernel waits for everybody's publish of that epoch).
//
// Consumers:
//   Krum               the Krum kernel (csrc/select.cu) reads the ranks' tables itself and writes the index to the device
//                      AND to mapped pinned host memory, so a Krum step ends with one stream synchronisation instead of
//                      a blocking 4-byte memcpy.
//   xgpu_sum_kernel    [wait] -> elementwise sum of the ranks' tables into a local table (Bulyan keeps its own selection
//                      kernels).
#include <string.h>

#include "afl_common.cuh"

namespace afl {
namespace gram {
int sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out, void* ws, size_t ws_bytes,
                   int flags, cudaStream_t stream);
}
namespace select {
int krum_tail(KrumParams p, int users_count, int corrupted_count, cudaStream_t stream, int batch = 1, bool rows = false);
}
namespace xgpu {

struct Ctx {
  int world, rank, n_max, device;
  size_t table_bytes, block_bytes;
  uint8_t* block;                       // own allocation
  uint8_t* peer[kMaxWorld];             // mapped blocks (peer[rank] == block)
  bool opened[kMaxWorld];
  unsigned long long epoch;
  float* score;                         // [n_max] local scratch
  int* idx_dev;                         // device copy of the last index
  int* idx_host;                        // mapped pinned host memory
  int* idx_host_devptr;
  int* status_host;                     // 0 ok, 1 = flag wait timed out
  int* status_host_devptr;
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
struct PublishParams { unsigned long long* flag[kMaxWorld]; int world, rank; unsigned long long epoch; };
__global__ void publish_kernel(const PublishParams p) {
  if (threadIdx.x < p.world) {
    __threadfence_system();                                              // the table written by earlier kernels of this stream
    st_release_sys(p.flag[threadIdx.x] + p.rank, p.epoch);
  }
}

struct SumParams { const double* tab[kMaxWorld]; const unsigned long long* flags; unsigned long long epoch; int world; size_t count; double* out; int* status_host; };
__global__ void __launch_bounds__(256)
xgpu_sum_kernel(const SumParams p) {
  if (!wait_flags(p.flags, p.world, p.epoch)) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *p.status_host = 1;
    return;
  }
  for (size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; e < p.count; e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    double s = 0.0;
    for (int r = 0; r < p.world; ++r) s += ld_peer_f64(p.tab[r] + e);
    p.out[e] = s;
  }
  if (threadIdx.x == 0 && blockIdx.x == 0) *p.status_host = 0;
}

static size_t flags_offset(const Ctx* c) { return 2 * c->table_bytes; }

int create(int world, int rank, int n_max, void** out) {
  if (!out || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || n_max < 1) { set_error("afl_xgpu_create: bad argument"); return AFL_ERR_BAD_ARG; }
  Ctx* c = new Ctx();
  memset(c, 0, sizeof(*c));
  c->world = world; c->rank = rank; c->n_max = n_max; c->device = current_device();
  c->table_bytes = align_up(static_cast<size_t>(n_max) * n_max * sizeof(double), 256);
  c->block_bytes = 2 * c->table_bytes + align_up(sizeof(unsigned long long) * kMaxWorld + 64, 256);
  AFL_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->block), c->block_bytes));
  AFL_CUDA(cudaMemset(c->block, 0, c->block_bytes));
  AFL_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->score), sizeof(float) * n_max + 256));
  AFL_CUDA(cudaMalloc(reinterpret_cast<void**>(&c->idx_dev), 256));
  AFL_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&c->idx_host), 64, cudaHostAllocMapped));
  AFL_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&c->idx_host_devptr), c->idx_host, 0));
  c->status_host = c->idx_host + 8;
  c->status_host_devptr = c->idx_host_devptr + 8;
  c->idx_host[0] = -1; c->status_host[0] = 0;
  c->peer[rank] = c->block; c->opened[rank] = false;
  AFL_CUDA(cudaDeviceSynchronize());
  *out = c;
  return AFL_OK;
}

int local_handle(void* ctx, unsigned char* out64) {
  Ctx* c = static_cast<Ctx*>(ctx);
  if (!c || !out64) { set_error("afl_xgpu_handle: bad argument"); return AFL_ERR_BAD_ARG; }
  cudaIpcMemHandle_t h;
  AFL_CUDA(cudaIpcGetMemHandle(&h, c->block));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(out64, &h, 64);
  return AFL_OK;
}

int connect(void* ctx, const unsigned char* handles) {
  Ctx* c = static_cast<Ctx*>(ctx);
  if (!c || !handles) { set_error("afl_xgpu_connect: bad argument"); return AFL_ERR_BAD_ARG; }
  for (int r = 0; r < c->world; ++r) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + static_cast<size_t>(r) * 64, 64);
    void* p = nullptr;
    AFL_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->peer[r] = static_cast<uint8_t*>(p);
    c->opened[r] = true;
  }
  return AFL_OK;
}

int destroy(void* ctx) {
  Ctx* c = static_cast<Ctx*>(ctx);
  if (!c) return AFL_OK;
  cudaDeviceSynchronize();
  for (int r = 0; r < c->world; ++r)
    if (c->opened[r]) cudaIpcCloseMemHandle(c->peer[r]);
  cudaFree(c->block); cudaFree(c->score); cudaFree(c->idx_dev); cudaFreeHost(c->idx_host);
  delete c;
  return AFL_OK;
}

static double* table_of(const Ctx* c, int r, unsigned long long epoch) {
  return reinterpret_cast<double*>(c->peer[r] + (epoch & 1ull) * c->table_bytes);
}

static int publish(Ctx* c, cudaStream_t stream) {
  if (c->world == 1) return AFL_OK;
  PublishParams pp{};
  for (int r = 0; r < c->world; ++r) pp.flag[r] = reinterpret_cast<unsigned long long*>(c->peer[r] + flags_offset(c));
  pp.world = c->world; pp.rank = c->rank; pp.epoch = c->epoch;
  publish_kernel<<<1, 32, 0, stream>>>(pp);
  AFL_LAUNCH_CHECK("publish_kernel");
  return AFL_OK;
}

// Whole sharded Krum step on this rank's [n, d_local] shard: partial table -> publish -> Krum kernel on the ranks'
// tables.  Enqueues only; *idx_host_out points to mapped pinned memory holding the index once `stream` has been
// synchronised.
int krum_step(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, int users_count, int corrupted_count,
              void* ws, size_t ws_bytes, int flags, cudaStream_t stream, int** idx_host_out, int** status_host_out,
              int** idx_dev_out) {
  Ctx* c = static_cast<Ctx*>(ctx);
  if (!c || n < 1 || n > c->n_max) { set_error("afl_krum_sharded: bad context or n > n_max"); return AFL_ERR_BAD_ARG; }
  if (c->device != current_device()) { set_error("afl_krum_sharded: context belongs to device %d", c->device); return AFL_ERR_BAD_ARG; }
  c->epoch += 1;
  double* mine = table_of(c, c->rank, c->epoch);
  int rc = gram::sqdist_partial(G, n, d, ld, dtype, mine, ws, ws_bytes, flags, stream);
  if (rc) return rc;
  rc = publish(c, stream);
  if (rc) return rc;
  KrumParams kp{};
  for (int r = 0; r < c->world; ++r) kp.tab[r] = table_of(c, r, c->epoch);
  kp.flags = reinterpret_cast<const unsigned long long*>(c->block + flags_offset(c));
  kp.epoch = c->epoch; kp.world = c->world; kp.n = n;
  kp.score = c->score;
  kp.done = reinterpret_cast<unsigned int*>(c->block + flags_offset(c) + sizeof(unsigned long long) * kMaxWorld);
  kp.idx_dev = c->idx_dev; kp.idx_host = c->idx_host_devptr; kp.status_host = c->status_host_devptr;
  rc = select::krum_tail(kp, users_count, corrupted_count, stream);
  if (rc) return rc;
  if (idx_host_out) *idx_host_out = c->idx_host;
  if (status_host_out) *status_host_out = c->status_host;
  if (idx_dev_out) *idx_dev_out = c->idx_dev;
  return AFL_OK;
}

// Partial table -> publish -> sum of all ranks' tables into d2_total (local device memory, n*n float64).
int sqdist_allreduce(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_total, void* ws,
                     size_t ws_bytes, int flags, cudaStream_t stream, int** status_host_out) {
  Ctx* c = static_cast<Ctx*>(ctx);
  if (!c || !d2_total || n < 1 || n > c->n_max) { set_error("afl_sqdist_allreduce: bad context or n > n_max"); return AFL_ERR_BAD_ARG; }
  if (c->device != current_device()) { set_error("afl_sqdist_allreduce: context belongs to device %d", c->device); return AFL_ERR_BAD_ARG; }
  if (c->world == 1) return gram::sqdist_partial(G, n, d, ld, dtype, d2_total, ws, ws_bytes, flags, stream);
  c->epoch += 1;
  int rc = gram::sqdist_partial(G, n, d, ld, dtype, table_of(c, c->rank, c->epoch), ws, ws_bytes, flags, stream);
  if (rc) return rc;
  rc = publish(c, stream);
  if (rc) return rc;
  SumParams sp{};
  for (int r = 0; r < c->world; ++r) sp.tab[r] = table_of(c, r, c->epoch);
  sp.flags = reinterpret_cast<const unsigned long long*>(c->block + flags_offset(c));
  sp.epoch = c->epoch; sp.world = c->world; sp.count = static_cast<size_t>(n) * n; sp.out = d2_total;
  sp.status_host = c->status_host_devptr;
  const size_t blocks = (sp.count + 255) / 256;
  {
    ProfScope ps("xgpu_sum", stream);
    xgpu_sum_kernel<<<static_cast<unsigned>(blocks > 592 ? 592 : blocks), 256, 0, stream>>>(sp);
  }
  AFL_LAUNCH_CHECK("xgpu_sum_kernel");
  if (status_host_out) *status_host_out = c->status_host;
  return AFL_OK;
}

}  // namespace xgpu
}  // namespace afl

using namespace afl;

extern "C" {
int afl_xgpu_create(int world, int rank, int n_max, void** ctx_out) { return xgpu::create(world, rank, n_max, ctx_out); }
int afl_xgpu_handle(void* ctx, unsigned char* out64) { return xgpu::local_handle(ctx, out64); }
int afl_xgpu_connect(void* ctx, const unsigned char* handles) { return xgpu::connect(ctx, handles); }
int afl_xgpu_destroy(void* ctx) { return xgpu::destroy(ctx); }
int afl_krum_sharded(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, int users_count, int corrupted_count,
                     void* workspace, size_t workspace_bytes, int flags, void* stream, int** idx_host_out,
                     int** status_host_out, int** idx_dev_out) {
  return xgpu::krum_step(ctx, G, n, d, ld, dtype, users_count, corrupted_count, workspace, workspace_bytes, flags,
                         static_cast<cudaStream_t>(stream), idx_host_out, status_host_out, idx_dev_out);
}
int afl_sqdist_allreduce(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_total, void* workspace,
                         size_t workspace_bytes, int flags, void* stream, int** status_host_out) {
  return xgpu::sqdist_allreduce(ctx, G, n, d, ld, dtype, d2_total, workspace, workspace_bytes, flags,
                                static_cast<cudaStream_t>(stream), status_host_out);
}
}
