// Krum (defences.py:23-42) and Bulyan's selection loop (defences.py:57-68) on an n x n distance table that is small
// enough (<= 64 MB of fp32 at n = 4096) to live in L2.  A batch of same-shape problems (consecutive tables) adds the
// problem to the grid: y for krum_tail_kernel and row_sort_kernel, x for bulyan_rounds_kernel.  A per-problem call
// (afl_defend_batched_each) also hands krum_tail_kernel and bulyan_rounds_kernel its ProblemParams table: each problem
// then reads its own take, or its own f and theta, instead of the scalar arguments.
//
//   krum_tail_kernel     one CTA per user u: u's n-1 distances -> bitonic sort in shared memory -> ascending sequential
//                        fp32 sum of the `take` smallest (defences.py:33-34) -> score[u]; the last CTA to finish does the
//                        strict-< argmin from (1e20, -1) in the dict order [1, 0, 2, ...] (defences.py:35-37).  The row
//                        is Sqdist (float64 d2 tables summed in rank order -> (float)sqrt(max(s, 0)), 32-bit keys) or Dist
//                        (a caller's fp32 table: 64-bit (|value|, neighbour) keys, the table's own values summed in that
//                        order, so a user-supplied table keeps the sign and NaN of its entries).
//   row_sort_kernel      Bulyan: one CTA per user sorts the user's n-1 distances (value, index) and emits the sorted
//                        values, the sorted neighbour indices and the inverse permutation (rank of every neighbour).
//   bulyan_rounds_kernel one persistent CTA per problem runs all theta rounds.  Removal of the selected user is an
//                        O(1) update per remaining user: its kept set (the m_r smallest alive distances)
//                        loses either the removed neighbour or its current largest kept element, tracked
//                        by a boundary pointer that only ever moves left over the pre-sorted row.  Scores
//                        are kept in float64, so every round's score is the exact sum of the fp32
//                        distances (the reference's fp32 sequential sum differs by rounding noise only).
#include <type_traits>

#include "afl_common.cuh"

namespace afl {
namespace select {

constexpr int kMaxN = 4096;

// Workspace of `batch` problems: Bulyan's sorted rows, or Krum's [last-CTA counters: batch, padded to 256 B][scores:
// batch x n floats].  Problem b's rows are at b * n * n in each array.
struct SortWs {
  float* sval;      // [batch][n][n]   sorted distances of row u (first n-1 entries valid)
  uint16_t* sidx;   // [batch][n][n]   neighbour index at each sorted position
  uint16_t* rank;   // [batch][n][n]   rank[u][v] = sorted position of neighbour v in row u
};

static size_t ws_bytes_for(int n, int batch) {
  const size_t nn = static_cast<size_t>(n) * n * batch;
  return align_up(nn * 4, 256) + 2 * align_up(nn * 2, 256) + align_up(static_cast<size_t>(n) * batch * 4, 256) + 256;
}

static SortWs carve(void* ws, int n, int batch) {
  const size_t nn = static_cast<size_t>(n) * n * batch;
  uint8_t* p = static_cast<uint8_t*>(ws);
  SortWs w;
  w.sval = reinterpret_cast<float*>(p); p += align_up(nn * 4, 256);
  w.sidx = reinterpret_cast<uint16_t*>(p); p += align_up(nn * 2, 256);
  w.rank = reinterpret_cast<uint16_t*>(p);
  return w;
}

// The reference's visit order [1, 0, 2, 3, ...]: position of user u, and (the map is its own inverse) user at position u.
__device__ __forceinline__ int visit_pos(int u) { return u == 1 ? 0 : (u == 0 ? 1 : u); }

// Ascending bitonic sort of keys[0, P), P a power of two, by the whole block.  The keys must be visible to the block.
template <typename Key>
__device__ __forceinline__ void block_bitonic_sort(Key* keys, int P) {
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const int lo = ((t / stride) * (stride << 1)) + (t % stride);
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const Key a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
}

// (score, visit position) order: strict < on the score, ties to the earlier-visited user.  Start from
// (+inf, 0x7fffffff) and feed only eligible scores (< 1e20, never NaN), so the minimum does not depend on the order.
template <typename T>
__device__ __forceinline__ void argmin_combine(T& best, int& best_pos, T v, int pos) {
  if (v < best || (v == best && pos < best_pos)) { best = v; best_pos = pos; }
}

// Block-wide argmin of every thread's (best, best_pos); kWarps = blockDim.x / 32.  Returns, in thread 0, the winning
// user or -1 when no thread saw an eligible score.
template <int kWarps, typename T>
__device__ __forceinline__ int block_argmin_user(T best, int best_pos) {
  __shared__ T s_val[kWarps];
  __shared__ int s_pos[kWarps];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmin_combine(best, best_pos, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, best_pos, o));
  if ((threadIdx.x & 31) == 0) { s_val[threadIdx.x >> 5] = best; s_pos[threadIdx.x >> 5] = best_pos; }
  __syncthreads();
  if (threadIdx.x >= 32) return -1;
  const bool have = threadIdx.x < kWarps;
  best = have ? s_val[threadIdx.x] : static_cast<T>(__int_as_float(0x7f800000));
  best_pos = have ? s_pos[threadIdx.x] : 0x7fffffff;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    argmin_combine(best, best_pos, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, best_pos, o));
  return best_pos == 0x7fffffff ? -1 : visit_pos(best_pos);
}

// Sort key of an fp32 distance: distances are >= 0 (or NaN), so the IEEE bit pattern orders like the value (NaN last);
// the neighbour in the low word keeps the sort stable.
__device__ __forceinline__ unsigned long long dist_key(float d, int v) {
  return (static_cast<unsigned long long>(__float_as_uint(d) & 0x7FFFFFFFu) << 32) | static_cast<unsigned>(v);
}

enum KrumSource { kSqdist, kDist };
template <KrumSource kSrc>
using KrumKey = typename std::conditional<kSrc == kSqdist, uint32_t, unsigned long long>::type;

template <KrumSource kSrc>
__device__ __forceinline__ KrumKey<kSrc> krum_key(const KrumParams& p, size_t off, int u, int v) {
  const size_t e = off + static_cast<size_t>(u) * p.n + v;
  if constexpr (kSrc == kSqdist) {
    double s = 0.0;
    for (int r = 0; r < p.world; ++r)                                    // fixed rank order: identical sum on every rank
      s += p.world > 1 ? ld_peer_f64(p.tab[r] + e) : p.tab[0][e];
    // defences.py:20 (np.float32 norm); a negative cancellation residue is 0, a NaN stays NaN (sorts last, never eligible)
    const float dist = static_cast<float>(sqrt(s > 0.0 ? s : (s == s ? 0.0 : s)));
    return __float_as_uint(dist) & 0x7FFFFFFFu;                          // >= 0 or NaN: the bit pattern orders like the value
  } else {
    return dist_key(p.dist[e], v);
  }
}

// The distance a sorted key stands for: the key itself, or the table's original bits (keeps a NaN a NaN).
template <KrumSource kSrc>
__device__ __forceinline__ float krum_value(const KrumParams& p, size_t off, int u, KrumKey<kSrc> k) {
  if constexpr (kSrc == kSqdist) return __uint_as_float(k);
  else return p.dist[off + static_cast<size_t>(u) * p.n + static_cast<int>(k & 0xFFFFFFFFu)];
}

// kRows (a ragged batch, afl_defend_batched_rows): problem b has m = each[b].tm.n_rows participating users in its n x n
// table (n stays the pitch).  CTAs u >= m only count themselves done, and the scores and the argmin cover users < m.
template <KrumSource kSrc, bool kRows>
__global__ void __launch_bounds__(256)
krum_tail_kernel(const KrumParams p) {
  using Key = KrumKey<kSrc>;
  extern __shared__ __align__(8) unsigned char smem[];
  Key* keys = reinterpret_cast<Key*>(smem);                              // P row keys
  __shared__ int s_last;
  const int u = blockIdx.x, n = p.n, b = blockIdx.y;                     // user u of problem b
  const size_t off = static_cast<size_t>(b) * n * n;
  float* score = p.score + static_cast<size_t>(b) * n;
  if constexpr (kSrc == kSqdist && !kRows) {                            // (a ragged batch is never a peer exchange)
    if (p.world > 1 && !wait_flags(p.flags, p.world, p.epoch)) {
      if (threadIdx.x == 0 && u == 0) { *p.status_host = 1; *p.idx_host = -1; *p.idx_dev = -1; }
      return;
    }
  }
  const int m = kRows ? p.each[b].tm.n_rows : n;
  const bool work = !kRows || u < m;
  if (work) {
    int P = 1;
    while (P < m) P <<= 1;
    for (int v = threadIdx.x; v < P; v += blockDim.x) keys[v] = (v < m && v != u) ? krum_key<kSrc>(p, off, u, v) : ~Key(0);
    __syncthreads();
    block_bitonic_sort(keys, P);
  }
  if (threadIdx.x == 0) {
    if (work) {
      float s = 0.f;                                                     // Python: sum() starts at int 0; ascending fp32 adds
      const int take = p.each ? p.each[b].take : p.take;
      for (int pos = 0; pos < take; ++pos) s = s + krum_value<kSrc>(p, off, u, keys[pos]);
      score[u] = s;
      __threadfence();
    }
    s_last = (atomicAdd(p.done + b, 1u) == static_cast<unsigned>(n - 1)) ? 1 : 0;
  }
  __syncthreads();
  if (!s_last) return;
  // ---- the last CTA: strict-< argmin from (1e20, -1) in the reference's visit order
  __threadfence();
  float best = __int_as_float(0x7f800000);
  int best_pos = 0x7fffffff;
  for (int v = threadIdx.x; v < m; v += blockDim.x) {
    const float s = __ldcg(score + v);
    if (m >= 2 && static_cast<double>(s) < 1e20) argmin_combine(best, best_pos, s, visit_pos(v));   // vs the Python float 1e20
  }
  const int idx = block_argmin_user<256 / 32>(best, best_pos);
  if (threadIdx.x == 0) {
    p.idx_dev[b] = idx;
    if (p.idx_host) { *p.idx_host = idx; *p.status_host = 0; }
    p.done[b] = 0u;                                                      // ready for the next step
    __threadfence_system();
  }
}

// Fills p.take and launches the kernel for the row source p selects, grid (n, batch).  p.done[0 .. batch) must be zero.
// rows: each problem's participating users are p.each[b].tm.n_rows (d2 tables only).
int krum_tail(KrumParams p, int users_count, int corrupted_count, cudaStream_t stream, int batch, bool rows) {
  p.take = krum_take(p.n, users_count, corrupted_count);
  int P = 1; while (P < p.n) P <<= 1;
  {
    ProfScope ps("krum_tail", stream);
    const dim3 grid(p.n, batch);
    if (p.dist) krum_tail_kernel<kDist, false><<<grid, 256, static_cast<size_t>(P) * sizeof(KrumKey<kDist>), stream>>>(p);
    else if (rows) krum_tail_kernel<kSqdist, true><<<grid, 256, static_cast<size_t>(P) * sizeof(KrumKey<kSqdist>), stream>>>(p);
    else krum_tail_kernel<kSqdist, false><<<grid, 256, static_cast<size_t>(P) * sizeof(KrumKey<kSqdist>), stream>>>(p);
  }
  AFL_LAUNCH_CHECK("krum_tail_kernel");
  return AFL_OK;
}

// kRows (a ragged batch): problem b sorts the first m = theta_b + 2 f_b entries of its rows u < m (n stays the pitch).
template <bool kRows>
__global__ void __launch_bounds__(256)
row_sort_kernel(const float* __restrict__ dist, int n, SortWs w, const ProblemParams* __restrict__ each) {
  extern __shared__ unsigned long long keys[];
  const int u = blockIdx.x;
  const int m = kRows ? each[blockIdx.y].theta + 2 * each[blockIdx.y].f : n;
  if (kRows && u >= m) return;
  const size_t off = static_cast<size_t>(blockIdx.y) * n * n;           // problem blockIdx.y
  dist += off; w.sval += off; w.sidx += off; w.rank += off;
  int P = 1;
  while (P < m) P <<= 1;
  for (int v = threadIdx.x; v < P; v += blockDim.x)
    keys[v] = (v < m && v != u) ? dist_key(dist[static_cast<size_t>(u) * n + v], v) : ~0ull;
  __syncthreads();
  block_bitonic_sort(keys, P);
  const size_t base = static_cast<size_t>(u) * n;
  for (int pos = threadIdx.x; pos < m; pos += blockDim.x) {
    const unsigned long long k = keys[pos];
    if (pos < m - 1) {
      const int v = static_cast<int>(k & 0xFFFFFFFFu);
      w.sval[base + pos] = dist[base + v];               // original bits (keeps a NaN a NaN)
      w.sidx[base + pos] = static_cast<uint16_t>(v);
      w.rank[base + v] = static_cast<uint16_t>(pos);
    } else {
      w.sval[base + pos] = 0.f;
      w.sidx[base + pos] = static_cast<uint16_t>(u);
      w.rank[base + u] = static_cast<uint16_t>(pos);
    }
  }
}

constexpr int kRowsPerThread = kMaxN / 1024;

// kRows (a ragged batch): problem b's users are u < m = theta_b + 2 f_b (its users_count); n stays the table pitch.
template <bool kRows>
__global__ void __launch_bounds__(1024, 1)
bulyan_rounds_kernel(const float* __restrict__ dist, int n, int f, int theta, SortWs w, int* __restrict__ sel_out,
                     const ProblemParams* __restrict__ each) {
  __shared__ uint8_t alive[kMaxN];
  __shared__ int s_winner;
  const size_t off = static_cast<size_t>(blockIdx.x) * n * n;           // one CTA per problem
  dist += off; w.sval += off; w.sidx += off; w.rank += off;
  sel_out += static_cast<size_t>(blockIdx.x) * theta;                    // with a table: theta = the longest problem's

  const int tid = threadIdx.x;
  if (each) {                                                            // this problem's f and rounds; -2: no such round
    const int theta_b = each[blockIdx.x].theta;
    for (int r = theta_b + tid; r < theta; r += 1024) sel_out[r] = -2;
    f = each[blockIdx.x].f; theta = theta_b;
  }
  const int m = kRows ? theta + 2 * f : n;
  double score[kRowsPerThread];
  int bptr[kRowsPerThread];

  for (int v = tid; v < kMaxN; v += 1024) alive[v] = (v < m) ? 1 : 0;
  // round 0: keep0 = min(m - f, m - 1) smallest distances, summed ascending in float64
  const int keep0 = min(m - f, m - 1);
#pragma unroll
  for (int r = 0; r < kRowsPerThread; ++r) {
    const int u = tid + r * 1024;
    score[r] = 0.0; bptr[r] = keep0 - 1;
    if (u < m) {
      const float* sv = w.sval + static_cast<size_t>(u) * n;
      double s = 0.0;
      for (int pos = 0; pos < keep0; ++pos) s += static_cast<double>(sv[pos]);
      score[r] = s;
    }
  }
  __syncthreads();

  for (int round = 0; round < theta; ++round) {
    // ---- argmin over alive users: (score, visit position), strict < with earliest-visited tie-break
    double best = __longlong_as_double(0x7ff0000000000000ll);
    int best_pos = 0x7fffffff;
#pragma unroll
    for (int r = 0; r < kRowsPerThread; ++r) {
      const int u = tid + r * 1024;
      if (u < m && alive[u] && score[r] < 1e20) argmin_combine(best, best_pos, score[r], visit_pos(u));
    }
    const int idx = block_argmin_user<1024 / 32>(best, best_pos);
    if (tid == 0) {
      s_winner = idx;
      sel_out[round] = idx;
      if (idx >= 0) alive[idx] = 0;
    }
    __syncthreads();
    const int s = s_winner;
    if (s < 0) {                       // nobody eligible (NaN / >= 1e20 scores): the reference raises here
      for (int r2 = round + 1 + tid; r2 < theta; r2 += 1024) sel_out[r2] = -1;
      return;
    }
    // ---- O(1) update of every surviving user's kept set: size shrinks by one each round
#pragma unroll
    for (int r = 0; r < kRowsPerThread; ++r) {
      const int u = tid + r * 1024;
      if (u < m && u != s && alive[u]) {
        const size_t base = static_cast<size_t>(u) * n;
        const int pos = w.rank[base + s];
        int b = bptr[r];
        if (b >= 0) {
          if (pos <= b) {
            score[r] -= static_cast<double>(dist[base + s]);
            if (pos == b) { do { --b; } while (b >= 0 && !alive[w.sidx[base + b]]); }
          } else {
            score[r] -= static_cast<double>(w.sval[base + b]);
            do { --b; } while (b >= 0 && !alive[w.sidx[base + b]]);
          }
          bptr[r] = b;
        }
      }
    }
    __syncthreads();
  }
}

int max_clients() { return kMaxN; }
size_t workspace_bytes(int n, int batch) { return ws_bytes_for(n < 1 ? 1 : n, batch < 1 ? 1 : batch); }
size_t workspace_bytes(int n) { return workspace_bytes(n, 1); }

static int check_ws(int n, int batch, void* ws, size_t ws_bytes) {
  if (n > kMaxN) { set_error("selection kernels support n <= %d clients (got %d)", kMaxN, n); return AFL_ERR_UNSUPPORTED; }
  if (!ws || ws_bytes < ws_bytes_for(n, batch) || (reinterpret_cast<uintptr_t>(ws) % 256) != 0) {
    set_error("selection workspace too small or misaligned (%zu < %zu)", ws_bytes, ws_bytes_for(n, batch));
    return AFL_ERR_WORKSPACE;
  }
  return AFL_OK;
}

// Krum on a workspace: the batch counters live at its start (cleared here: workspaces are not initialised), the
// scores behind them unless the caller wants them.
static int krum_on_workspace(KrumParams p, int batch, int users_count, int corrupted_count, float* scores_out, void* ws,
                             size_t ws_bytes, cudaStream_t stream, bool rows = false) {
  int rc = check_ws(p.n, batch, ws, ws_bytes);
  if (rc) return rc;
  p.done = static_cast<unsigned int*>(ws);
  p.score = scores_out ? scores_out
                       : reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + align_up(static_cast<size_t>(batch) * 4, 256));
  AFL_CUDA(cudaMemsetAsync(p.done, 0, static_cast<size_t>(batch) * sizeof(unsigned int), stream));
  return krum_tail(p, users_count, corrupted_count, stream, batch, rows);
}

int krum_select(const float* dist, int n, int users_count, int corrupted_count, int* idx_out, float* scores_out,
                void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (!dist || !idx_out || n < 1) { set_error("afl_krum_select: bad argument"); return AFL_ERR_BAD_ARG; }
  KrumParams p{};
  p.dist = dist; p.n = n; p.idx_dev = idx_out;
  return krum_on_workspace(p, 1, users_count, corrupted_count, scores_out, ws, ws_bytes, stream);
}

// d2: batch consecutive n x n tables; idx_out[batch]; each (device, may be NULL): per-problem take, and with rows also
// the problem's participating users (tm.n_rows)
int krum_from_sqdist(const double* d2, int n, int users_count, int corrupted_count, int* idx_out, void* ws,
                     size_t ws_bytes, cudaStream_t stream, int batch, const ProblemParams* each, bool rows) {
  if (!d2 || !idx_out || n < 1 || (rows && !each)) { set_error("afl_krum_from_sqdist: bad argument"); return AFL_ERR_BAD_ARG; }
  KrumParams p{};
  p.tab[0] = d2; p.world = 1; p.n = n; p.idx_dev = idx_out; p.each = each;
  return krum_on_workspace(p, batch, users_count, corrupted_count, nullptr, ws, ws_bytes, stream, rows);
}

int bulyan_rounds(const float* dist, int n, int f, int theta, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream, int batch, const ProblemParams* each, bool rows);

// dist: batch consecutive n x n tables; sel_out[batch][theta], theta = users_count - 2f.  each (device, may be NULL):
// per-problem f and theta; f is then the smallest problem's, so that every row of sel_out holds its problem's rounds.
int bulyan_select(const float* dist, int n, int users_count, int f, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream, int batch, const ProblemParams* each) {
  if (!dist || !sel_out || n < 1 || f < 0) { set_error("afl_bulyan_select: bad argument"); return AFL_ERR_BAD_ARG; }
  if (users_count < 4 * f + 3) {
    set_error("bulyan: users_count >= 4*corrupted_count + 3 violated (%d, %d)", users_count, f);
    return AFL_ERR_PRECONDITION;
  }
  if (users_count != n) {
    set_error("afl_bulyan_select: users_count (%d) must equal the number of rows (%d)", users_count, n);
    return AFL_ERR_UNSUPPORTED;
  }
  return bulyan_rounds(dist, n, f, users_count - 2 * f, sel_out, ws, ws_bytes, stream, batch, each, false);
}

// The two Bulyan kernels on checked arguments: sel_out[batch][theta].  rows (a ragged batch, each required): problem b's
// users are each[b].theta + 2 each[b].f of its n x n table.
int bulyan_rounds(const float* dist, int n, int f, int theta, int* sel_out, void* ws, size_t ws_bytes,
                  cudaStream_t stream, int batch, const ProblemParams* each, bool rows) {
  int rc = check_ws(n, batch, ws, ws_bytes);
  if (rc) return rc;
  const SortWs w = carve(ws, n, batch);
  int P = 1; while (P < n) P <<= 1;
  const dim3 grid(n, batch);
  const size_t smem = static_cast<size_t>(P) * sizeof(unsigned long long);
  {
    ProfScope ps("row_sort", stream);
    if (rows) row_sort_kernel<true><<<grid, 256, smem, stream>>>(dist, n, w, each);
    else row_sort_kernel<false><<<grid, 256, smem, stream>>>(dist, n, w, nullptr);
  }
  AFL_LAUNCH_CHECK("row_sort_kernel");
  ProfScope ps("bulyan_rounds", stream);
  if (rows) bulyan_rounds_kernel<true><<<batch, 1024, 0, stream>>>(dist, n, f, theta, w, sel_out, each);
  else bulyan_rounds_kernel<false><<<batch, 1024, 0, stream>>>(dist, n, f, theta, w, sel_out, each);
  AFL_LAUNCH_CHECK("bulyan_rounds_kernel");
  return AFL_OK;
}

}  // namespace select
}  // namespace afl
