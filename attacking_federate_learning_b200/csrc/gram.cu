// Pairwise squared distances of the N client rows (reference: defences.py:16-21
// `_krum_create_distances`, the dominant cost of Krum and Bulyan).
//
// Tensor-core path (fp32, bf16 or fp16 input, 16-byte aligned rows): d2_ij = s_ii + s_jj - 2 s_ij with S = G G^T on the
// Hopper warpgroup MMAs (csrc/gram_pair.cu), fp32 split into two bf16 or two TF32 terms, 16-bit clients as they are, K split over CTAs and the
// partial tiles summed in a fixed order in float64 -> bit-reproducible, and identical rows give exact zeros and
// bit-identical table rows outside the rows between them (Krum's [1,0,2,...] tie-break relies on this; DESIGN 2.1).
//
// SIMT path (any pitch, fp32, bf16 or fp16): direct sum of squared fp32 differences, float64 accumulation.
// Used for misaligned pitches and as an independent check of the tensor path in the tests.
#include "afl_common.cuh"

namespace afl {
namespace gram {

// ------------------------------------------------------------------------------------------------
// SIMT difference kernel: block = 16x16 threads, tile = 32 x 32 client pairs, k-chunks of 32.
// ------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float load_elem(const T* p);
template <> __device__ __forceinline__ float load_elem<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float load_elem<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}
template <> __device__ __forceinline__ float load_elem<__half>(const __half* p) { return __half2float(*p); }

// blockIdx.z = problem of a batch (matrix at G + z * batch_stride, partials at part + z * splits * n * n).
template <typename T>
__global__ void __launch_bounds__(256)
sqdist_simt_kernel(const T* __restrict__ G, int n, int64_t d, int64_t ld, int64_t batch_stride, int splits,
                   double* __restrict__ part) {
  __shared__ float As[32][33], Bs[32][33];
  const int tiles = (n + 31) / 32;
  const int ti = blockIdx.x / tiles, tj = blockIdx.x % tiles;
  if (tj > ti) return;                                  // lower triangle (incl. diagonal tiles)
  const int split = blockIdx.y;
  G += blockIdx.z * batch_stride;
  part += static_cast<size_t>(blockIdx.z) * splits * n * n;
  const int64_t chunks = (d + 31) / 32;
  const int64_t c0 = chunks * split / splits, c1 = chunks * (split + 1) / splits;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[2][2] = {{0, 0}, {0, 0}};
  for (int64_t c = c0; c < c1; ++c) {
    const int64_t col0 = c * 32;
    for (int e = threadIdx.x; e < 32 * 32; e += 256) {
      const int r = e >> 5, k = e & 31;
      const int64_t col = col0 + k;
      const int ra = ti * 32 + r, rb = tj * 32 + r;
      As[r][k] = (ra < n && col < d) ? load_elem<T>(G + static_cast<int64_t>(ra) * ld + col) : 0.f;
      Bs[r][k] = (rb < n && col < d) ? load_elem<T>(G + static_cast<int64_t>(rb) * ld + col) : 0.f;
    }
    __syncthreads();
    float part32[2][2] = {{0, 0}, {0, 0}};
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
          const float df = As[ty * 2 + u][k] - Bs[tx * 2 + v][k];   // fl32(g_i - g_j), as the reference
          part32[u][v] = fmaf(df, df, part32[u][v]);
        }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
      for (int v = 0; v < 2; ++v) acc[u][v] += static_cast<double>(part32[u][v]);
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const int i = ti * 32 + ty * 2 + u, j = tj * 32 + tx * 2 + v;
      if (i < n && j < n && j < i) part[(static_cast<size_t>(split) * n + i) * n + j] = acc[u][v];
    }
}

__global__ void sqdist_simt_reduce_kernel(const double* __restrict__ part, int n, int splits,
                                          double* __restrict__ d2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= n) return;
  part += static_cast<size_t>(blockIdx.z) * splits * n * n;   // problem blockIdx.z
  d2 += static_cast<size_t>(blockIdx.z) * n * n;
  double v = 0.0;
  if (i != j) {
    const int hi = max(i, j), lo = min(i, j);
    for (int s = 0; s < splits; ++s) v += part[(static_cast<size_t>(s) * n + hi) * n + lo];
  }
  d2[static_cast<size_t>(i) * n + j] = v;
}

// `total` = batch * n * n: the tables of a batch are consecutive
__global__ void sqdist_to_dist_kernel(const double* __restrict__ d2, int n, size_t total, float* __restrict__ dist) {
  const size_t e = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const size_t r = e % (static_cast<size_t>(n) * n);
  const int i = static_cast<int>(r / n), j = static_cast<int>(r % n);
  const double v = d2[e];
  // a negative cancellation residue is 0; NaN (two SIMT rows with the same infinity in one column) stays NaN
  dist[e] = (i == j) ? 0.f : static_cast<float>(sqrt(v > 0.0 ? v : (v == v ? 0.0 : v)));
}

// tensor-core tile-pair kernel (gram_pair.cu)
size_t pair_parts_bytes(int n, int64_t d, int batch);
size_t pair_center_bytes(int64_t d, int batch);
int launch_pair(const void* G, int mode, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, float* parts,
                double* S, float* cvec, double* d2_out, int flush, int center, int single_pass, cudaStream_t stream,
                const ProblemParams* rows);

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct Plan {
  bool tensor;
  int mode;           // GramMode of the tensor-core kernel
  int simt_splits;
  size_t parts_bytes, s_bytes, total;
};

static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}

// batch > 1 adds the batch pitch to the alignment TMA needs, and a pitch that keeps the problems apart (the 3-D tensor map)
static bool tensor_eligible(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype) {
  const int64_t per16 = dtype == AFL_F32 ? 4 : 8;           // elements per 16 bytes: TMA needs 16-byte aligned rows
  return (dtype == AFL_F32 || dtype == AFL_BF16 || dtype == AFL_F16) && (ld % per16 == 0) && (reinterpret_cast<uintptr_t>(G) % 16 == 0) && n >= 1 &&
         d >= 1 && n <= 4096 && d < (int64_t(1) << 31) - 64 &&
         (batch == 1 || (batch_stride % per16 == 0 && batch_stride >= static_cast<int64_t>(n) * ld));
}

// fp32 operands default to the centred bf16x2 split for N > 128 and for the streaming shapes (64 <= N_pad <= 112,
// D >= 32768); elsewhere, and with AFL_GRAM_TF32X2 / AFL_GRAM_SINGLE_PASS, to the split-TF32 operands (smaller
// uniform bias, no centring).  bf16 and fp16 clients are the operands themselves (kModeBf16In, kModeF16In); the fp32
// operand flags do not apply to them.  A batch chooses like one problem of its shape; its split counts see batch times
// the CTAs of one problem, and AFL_GRAM_SPLITS overrides both paths' split count.  A multi-tile bf16x2 batch holds one
// centre vector per problem.
static Plan make_plan(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, int flags) {
  Plan pl{};
  pl.tensor = !(flags & AFL_GRAM_FORCE_SIMT) && tensor_eligible(G, batch, batch_stride, n, d, ld, dtype);
  const int sms = sm_count();
  if (pl.tensor) {
    const int nb = (n + 15) & ~15;
    const bool streaming = nb >= 64 && nb <= 112 && d >= 32768;
    if (dtype == AFL_BF16) pl.mode = kModeBf16In;
    else if (dtype == AFL_F16) pl.mode = kModeF16In;
    else if ((flags & (AFL_GRAM_SINGLE_PASS | AFL_GRAM_TF32X2)) || !(n > 128 || streaming)) pl.mode = kModeTf32x2;
    else pl.mode = kModeBf16x2;
    pl.parts_bytes = pair_parts_bytes(n, d, batch);
    pl.s_bytes = align_up(static_cast<size_t>(batch) * n * n * sizeof(double), 256);
    pl.total = pl.parts_bytes + pl.s_bytes + pair_center_bytes(d, pl.mode == kModeBf16x2 && n > 128 ? batch : 1);
  } else {
    const int t32 = (n + 31) / 32;
    int64_t chunks = (d + 31) / 32;
    int s = (sms * 8) / (t32 * (t32 + 1) / 2 * batch); if (s < 1) s = 1;
    if (env_int("AFL_GRAM_SPLITS", 0) > 0) s = env_int("AFL_GRAM_SPLITS", 0);
    if (s > chunks) s = static_cast<int>(chunks);
    if (s > 1024) s = 1024;
    pl.simt_splits = s;
    pl.total = static_cast<size_t>(s) * batch * n * n * sizeof(double);
  }
  pl.total = align_up(pl.total, 256);
  return pl;
}

size_t workspace_bytes(int n, int64_t d, int dtype, int flags, int batch) {
  // Upper bound that holds for either path (the pointer alignment is unknown here).
  Plan a = make_plan(reinterpret_cast<const void*>(16), batch, static_cast<int64_t>(n) * 8, n, d, 8, dtype, flags & ~AFL_GRAM_FORCE_SIMT);
  Plan b = make_plan(reinterpret_cast<const void*>(16), batch, static_cast<int64_t>(n) * 8, n, d, 8, dtype, flags | AFL_GRAM_FORCE_SIMT);
  return (a.total > b.total ? a.total : b.total) + 256;
}

// `batch` problems of the same shape, problem b at G + b * batch_stride elements; d2_out: batch consecutive n x n tables.
// One problem is batch = 1 (batch_stride unused).  rows (device, may be NULL): a ragged batch's table; problem b's rows
// past rows[b].tm.n_rows then affect only the table entries that involve them.
int sqdist_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype, double* d2_out,
                   void* ws, size_t ws_bytes, int flags, cudaStream_t stream, const ProblemParams* rows) {
  if (!G || !d2_out || n < 1 || d < 1 || ld < d) { set_error("afl_sqdist_partial: bad argument"); return AFL_ERR_BAD_ARG; }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_sqdist_partial: dtype"); return AFL_ERR_UNSUPPORTED; }
  Plan pl = make_plan(G, batch, batch_stride, n, d, ld, dtype, flags);
  if ((flags & AFL_GRAM_FORCE_TCGEN05) && !pl.tensor) {
    set_error("afl_sqdist_partial: tensor-core path needs a 16-byte aligned base, 16-byte aligned pitch, n <= 4096");
    return AFL_ERR_UNSUPPORTED;
  }
  if (!ws || ws_bytes < pl.total || (reinterpret_cast<uintptr_t>(ws) % 256) != 0) {
    set_error("afl_sqdist_partial: workspace too small or misaligned (%zu < %zu)", ws_bytes, pl.total);
    return AFL_ERR_WORKSPACE;
  }
  const dim3 rblock(128), rgrid((n + 127) / 128, n, batch);
  if (pl.tensor) {
    // translation invariance: bf16x2 operands are converted as g - (mean of the last 8 clients) unless switched off
    const int center = !(flags & AFL_GRAM_NO_CENTER) && env_int("AFL_GRAM_CENTER", 1) != 0;
    float* parts = static_cast<float*>(ws);
    double* S = reinterpret_cast<double*>(static_cast<uint8_t*>(ws) + pl.parts_bytes);
    float* cvec = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + pl.parts_bytes + pl.s_bytes);
    return launch_pair(G, pl.mode, batch, batch_stride, n, d, ld, parts, S, cvec, d2_out, env_int("AFL_GRAM_FLUSH", 4),
                       center, (flags & AFL_GRAM_SINGLE_PASS) ? 1 : 0, stream, rows);
  } else {
    const int t32 = (n + 31) / 32;
    double* part = static_cast<double*>(ws);
    const dim3 grid(t32 * t32, pl.simt_splits, batch);
    {
      ProfScope ps("sqdist_simt", stream);
      if (dtype == AFL_F32)
        sqdist_simt_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(G), n, d, ld, batch_stride,
                                                            pl.simt_splits, part);
      else if (dtype == AFL_BF16)
        sqdist_simt_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(static_cast<const __nv_bfloat16*>(G), n, d, ld,
                                                                     batch_stride, pl.simt_splits, part);
      else
        sqdist_simt_kernel<__half><<<grid, 256, 0, stream>>>(static_cast<const __half*>(G), n, d, ld, batch_stride,
                                                              pl.simt_splits, part);
    }
    AFL_LAUNCH_CHECK("sqdist_simt_kernel");
    sqdist_simt_reduce_kernel<<<rgrid, rblock, 0, stream>>>(part, n, pl.simt_splits, d2_out);
    AFL_LAUNCH_CHECK("sqdist_simt_reduce_kernel");
  }
  return AFL_OK;
}

size_t workspace_bytes(int n, int64_t d, int dtype, int flags) { return workspace_bytes(n, d, dtype, flags, 1); }

int sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out, void* ws, size_t ws_bytes,
                   int flags, cudaStream_t stream) {
  return sqdist_batched(G, 1, 0, n, d, ld, dtype, d2_out, ws, ws_bytes, flags, stream, nullptr);
}

// batch consecutive n x n tables
int sqdist_to_dist(const double* d2, int n, float* dist, cudaStream_t stream, int batch) {
  if (!d2 || !dist || n < 1) { set_error("afl_sqdist_to_dist: bad argument"); return AFL_ERR_BAD_ARG; }
  const size_t total = static_cast<size_t>(batch) * n * n;
  sqdist_to_dist_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(d2, n, total, dist);
  AFL_LAUNCH_CHECK("sqdist_to_dist_kernel");
  return AFL_OK;
}

}  // namespace gram
}  // namespace afl
