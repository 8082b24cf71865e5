/*
 * afl_b200.h — C ABI of the GPU-native (H100, sm_90a) Byzantine-robust aggregation engine.
 *
 * The upstream reference (shaneson0/attacking_federate_learning) has no FFI: its boundary for this
 * path is a Python dict of callables, `defences.defend[name](users_grads, users_count,
 * corrupted_count)` (defences.py:73-75, called from server.py:87), plus the template-method class
 * `malicious.Attack` (malicious.py:4-36, called from main.py:67-68).  Each entry point below states
 * the reference function (file:line) whose arithmetic it replaces.  The Python mirror of the
 * reference interface (attacking_federate_learning_b200/defences.py, malicious.py) binds these
 * symbols with ctypes; INTEGRATION.md shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - Every function returns an afl_status (0 = ok).  Nothing throws across the ABI.
 *     afl_last_error() returns a thread-local, human-readable description of the last failure.
 *   - "device" pointers are CUDA device pointers on the current device; "host" pointers are plain
 *     host memory (pinned or pageable).  `stream` is a cudaStream_t passed as void* (NULL = legacy
 *     default stream).  Device entry points only enqueue work; they never synchronise.
 *   - Matrices are row-major `[n rows = clients][d columns = parameters]`, `ld` = row pitch in
 *     ELEMENTS (server.py:35 allocates users_grads as a C-contiguous N x D fp32 array, ld == d).
 *   - dtype of a device client matrix: AFL_F32 (the reference's only type), AFL_BF16 (config
 *     "trimmed_mean, bf16") or AFL_F16 (fp16 client updates, as sent over the uplink or produced by
 *     `.half()` models).  A 16-bit matrix computes the reference's result on its values upcast to fp32
 *     (exact); outputs are always fp32.  Any other code is AFL_ERR_UNSUPPORTED.  The host-buffer entry
 *     points take fp32 only.
 *   - No entry point allocates device memory; scratch comes from a caller-owned workspace whose size
 *     the matching *_workspace_bytes() function reports.
 *   - Multi-GPU: the parameter dimension D is sharded; every GPU calls the same entry points on its
 *     own `[n, d_local]` shard.  The only exchange is a sum-all-reduce of the n x n float64 table
 *     produced by afl_sqdist_partial() (done by the host layer over NCCL) before
 *     afl_sqdist_to_dist().
 */
#ifndef AFL_B200_H_
#define AFL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum afl_status {
  AFL_OK = 0,
  AFL_ERR_BAD_ARG = 1,       /* null pointer, negative size, misaligned buffer ...               */
  AFL_ERR_PRECONDITION = 2,  /* the reference's `assert` would fire (n >= 2f+1, n >= 4f+3)         */
  AFL_ERR_CUDA = 3,          /* a CUDA call failed; see afl_last_error()                          */
  AFL_ERR_UNSUPPORTED = 4,   /* dtype / size outside what the kernels implement                   */
  AFL_ERR_WORKSPACE = 5,     /* workspace too small                                               */
  AFL_ERR_NO_WINNER = 6,     /* a Bulyan round found no eligible user (NaN / >= 1e20 scores): the      */
                             /* reference raises KeyError(-1) at defences.py:66 (`distances.pop(-1)`)  */
  AFL_ERR_NAN_LOSS = 7,      /* backdoor training: the minibatch loss is NaN ("Got nan loss")         */
  AFL_ERR_NAN_DIST_LOSS = 8  /* backdoor training: the distance loss is NaN ("Got nan dist loss")     */
} afl_status;

typedef enum afl_dtype { AFL_F32 = 0, AFL_BF16 = 1, AFL_F16 = 2 } afl_dtype;

/* flags for afl_sqdist_partial */
enum {
  AFL_GRAM_AUTO = 0,          /* tensor-core (wgmma) path when the layout allows TMA, otherwise SIMT */
  AFL_GRAM_FORCE_SIMT = 1,    /* CUDA-core difference kernel (verification / unaligned pitch)      */
  AFL_GRAM_FORCE_TCGEN05 = 2, /* fail with AFL_ERR_UNSUPPORTED instead of falling back to SIMT     */
  AFL_GRAM_SINGLE_PASS = 4,   /* tensor path: hi*hi only (plain TF32), for measurement              */
  AFL_GRAM_TF32X2 = 16,       /* tensor path: split-TF32 operands for fp32 input (the default when N <= 128 outside */
                              /* the bf16x2 range below)                                            */
  AFL_GRAM_BF16X2 = 32,       /* accepted, ignored: fp32 input gets centred bf16x2 operands by default when N > 128 */
                              /* or 64 <= N_pad <= 112 and D >= 32768                                */
  AFL_GRAM_NO_CENTER = 64,    /* bf16x2 operands: do not subtract the last client's row while converting (the  */
                              /* default makes the table translation invariant; env AFL_GRAM_CENTER=0 too)    */
  AFL_GRAM_REWRITE_HI = 8     /* accepted, ignored (the split-TF32 converter always writes hi = the   */
                              /* fp32 operand with its low 13 mantissa bits cleared)                 */
};

/* ---- library / device ------------------------------------------------------------------------ */
const char* afl_version(void);
const char* afl_last_error(void);
/* Number of SMs, compute capability and free/total HBM bytes of the current device. */
int afl_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* free_bytes, size_t* total_bytes);
/* Number of kernel launches this library has issued since load (all threads). */
uint64_t afl_launch_count(void);

/* ---- in-library kernel timing (measurement aid for bench.py) -----------------------------------
 * While enabled, the dominant kernel of every entry point is bracketed by CUDA events on the stream it
 * is launched on.  afl_profile_read(name, ...) waits for the recorded events of kernel `name`
 * ("gram_pair", "sqdist_simt", "trimmed_mean", "alie", "mean", "krum_tail", "row_sort", "bulyan_rounds",
 * "honest_deviation"), returns their summed duration and launch count, and forgets them.  on = 1: every bracketed kernel; on = 2: only the
 * dominant kernel of a rule (gram_pair, sqdist_simt, trimmed_mean, mean, alie) - one pair of events per step. */
int afl_profile_enable(int on);
int afl_profile_read(const char* kernel, double* total_ms, int* launches);

/* ---- plain mean:  defences.py:13-14  no_defense -> np.mean(users_grads, axis=0) --------------- */
int afl_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, void* stream);

/* ---- pairwise squared distances:  defences.py:16-21  _krum_create_distances ------------------- */
/* Partial squared L2 distances over this shard's d columns, as a dense symmetric n x n float64
 * table (zero diagonal).  AFL_GRAM_AUTO: G*G^T on the tensor cores (wgmma, TMA-fed, bf16x2 or split-TF32
 * operands for fp32, bf16 and fp16 as they are; lower-triangular 128 x 128 tile pairs), d2_ij = s_ii + s_jj - 2 s_ij, bf16x2
 * operands centred on the mean of the last 8 clients' rows.  Partial tables of different shards
 * ADD; take the square root only after the all-reduce (afl_sqdist_to_dist). */
size_t afl_sqdist_workspace_bytes(int n, int64_t d, int dtype, int flags);
int afl_sqdist_partial(const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_out,
                       void* workspace, size_t workspace_bytes, int flags, void* stream);
/* dist[i][j] = (float)sqrt(max(d2[i][j], 0)), zero diagonal — the values the reference keeps in its
 * dict-of-dicts (np.float32 scalars, defences.py:20). */
int afl_sqdist_to_dist(const double* d2, int n, float* dist, void* stream);

/* ---- Krum selection:  defences.py:23-42  krum(..., return_index=True) --------------------------
 * score(u) = sum of the (users_count - corrupted_count) smallest of u's n-1 distances (ascending
 * fp32 sequential sum, like Python's sum(sorted(...)[:m])); strict-< argmin from (1e20, -1) visiting
 * users in the reference's dict order [1, 0, 2, 3, ...].  *idx_out (device int) receives the index
 * or -1.  scores_out (device float[n]) may be NULL.  No precondition check here: like the reference,
 * the `users_count >= 2f+1` assert belongs to the caller that wants the row (afl_krum). */
size_t afl_select_workspace_bytes(int n);
int afl_krum_select(const float* dist, int n, int users_count, int corrupted_count, int* idx_out,
                    float* scores_out, void* workspace, size_t workspace_bytes, void* stream);

/* The same selection straight from an (all-reduced) squared-distance table d2 (device float64[n*n]): the
 * distances are (float)sqrt(max(d2, 0)) as in afl_sqdist_to_dist, computed inside the Krum kernel, so the
 * index equals afl_krum_select(afl_sqdist_to_dist(d2)).  One call per aggregation after the all-reduce. */
int afl_krum_from_sqdist(const double* d2, int n, int users_count, int corrupted_count, int* idx_out,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ---- Bulyan selection:  defences.py:57-68 ------------------------------------------------------
 * theta = users_count - 2f rounds of Krum-with-removal on one distance table; sel_out (device
 * int[theta]) receives the indices in selection order.  Returns AFL_ERR_PRECONDITION unless
 * users_count >= 4f+3 (defences.py:56). */
int afl_bulyan_select(const float* dist, int n, int users_count, int corrupted_count, int* sel_out,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- trimmed mean around the median:  defences.py:44-52  trimmed_mean --------------------------
 * Per column: med = median (even count -> fl32 mean of the two middle values); keep the
 * k = rows - corrupted_count - 1 values with the smallest |fl32(x - med)| (ties: earlier row first);
 * out = mean(kept deviations) + med.  `row_index` (device int[n_rows], may be NULL = rows 0..n-1)
 * selects and ORDERS the participating rows — Bulyan's second stage passes its selection sequence
 * here so the theta x D gather of defences.py:70 is never materialised. */
int afl_trimmed_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index,
                     int n_rows, int corrupted_count, float* out, void* stream);

/* ---- gather one row chosen on the device (Krum's result as a dense vector) --------------------- */
int afl_gather_row(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* idx_dev,
                   float* out, void* stream);

/* ---- ALIE attack:  malicious.py:10-27,34-36  Attack.attack + DriftAttack._attack_grads ---------
 * Over the f malicious rows: mu = mean, sigma = sqrt(population variance); crafted = mu - z*sigma.
 * mu_out receives the UNPERTURBED mean when crafted_out != mu_out; pass crafted_out == mu_out to
 * reproduce the reference's in-place `grads_mean[:] -= z*stdev` aliasing.  If bcast_rows != NULL the
 * crafted vector is also written into rows 0..f-1 of that fp32 matrix (pitch bcast_ld), which is
 * what server.py:82-83 does next with the f aliased `usr.grads`. */
int afl_alie(const void* G_mal, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out,
             float* sigma_out, float* crafted_out, float* bcast_rows, int64_t bcast_ld, void* stream);

/* ---- ALIE band:  malicious.py:35 (x == NULL)  and  backdoor.py:60-61 (x != NULL) --------------
 * lo = mu - z*sigma, hi = mu + z*sigma in fp32 (the roundings of `grads_mean -/+ num_std*grads_stdev`).
 * x == NULL: out = lo, DriftAttack._attack_grads on statistics that already exist on the device.
 * x != NULL: out = np.clip(x, lo, hi) (NaN propagates as in NumPy), the clamp BackdoorAttack applies to
 * the gradient its maliciously trained network asks for.  fp32 device vectors of length d; out may
 * alias mu or x. */
int afl_alie_band(const float* mu, const float* sigma, double z, const float* x, float* out, int64_t d,
                  void* stream);

/* ---- server momentum step:  server.py:89-90 ----------------------------------------------------
 * v = momentum*v - lr*g ;  w += v   (fp32, in place). */
int afl_momentum_step(float* weights, float* velocity, const float* grads, int64_t d, float momentum,
                      float learning_rate, void* stream);
/* afl_momentum_step on `batch` contiguous rows of d floats (weights, velocity and grads: device fp32 [batch][d]), row b
 * at its own learning rate learning_rate[b] (device fp32 [batch], read when the kernel runs) in one launch: row b's
 * bits equal afl_momentum_step's at learning_rate[b].  A NULL pointer, batch < 1 or d < 1 -> AFL_ERR_BAD_ARG;
 * batch > 65535 -> AFL_ERR_UNSUPPORTED. */
int afl_momentum_step_batched(float* weights, float* velocity, const float* grads, int batch, int64_t d,
                              float momentum, const float* learning_rate, void* stream);

/* ---- multi-GPU exchange over NVLink peer memory (SURVEY 8e: "exactly one sum of the n x n partial table") ------
 * One process per GPU.  Every rank creates a context, exports its 64-byte CUDA IPC handle, the host layer gathers
 * the handles of all ranks (any transport) and every rank maps its peers.  world == 1 needs no connect.
 *   afl_krum_sharded     partial table of this rank's [n, d_local] shard (afl_sqdist_partial) -> published to the peers ->
 *                        fused tail: sum of the ranks' tables in rank order, sqrt, per-client sort, Krum score, argmin
 *                        (defences.py:16-42).  Enqueues only.  After `stream` is synchronised *idx_host_out (mapped
 *                        pinned memory) holds the index (identical on every rank), *status_host_out is 0 (1: a peer did
 *                        not publish in time) and *idx_dev_out is the device copy (for afl_gather_row).
 *   afl_sqdist_allreduce the same exchange, result = the summed table in d2_total (device, n*n float64) for callers
 *                        that run their own selection (Bulyan). */
int afl_xgpu_create(int world, int rank, int n_max, void** ctx_out);
int afl_xgpu_handle(void* ctx, unsigned char* out64);
int afl_xgpu_connect(void* ctx, const unsigned char* handles /* world x 64 bytes, rank order */);
int afl_xgpu_destroy(void* ctx);
int afl_krum_sharded(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, int users_count, int corrupted_count,
                     void* workspace, size_t workspace_bytes, int flags, void* stream, int** idx_host_out,
                     int** status_host_out, int** idx_dev_out);
int afl_sqdist_allreduce(void* ctx, const void* G, int n, int64_t d, int64_t ld, int dtype, double* d2_total, void* workspace,
                         size_t workspace_bytes, int flags, void* stream, int** status_host_out);

/* ---- one-call host-buffer API (what a cgo/ctypes binding of server.py:87 would call) ----------
 * rule: "NoDefense" | "Krum" | "TrimmedMean" | "Bulyan" (defences.py:4-8).  G_host: n x d fp32 in
 * host memory, pitch ld.  The call streams column slabs through a bounded device staging area (H2D
 * copies overlap the kernels), runs the rule, and writes the aggregated gradient to out_host[d] (fp32)
 * and, for Krum, the winning index to *idx_out (may be NULL).  Blocking.  Reference assert failures
 * map to AFL_ERR_PRECONDITION.  `slab_cols` = columns per staging slab (0 = default, about 96 MB).
 * The matrix does not have to fit the GPU: Krum, TrimmedMean and NoDefense stream every slab through a
 * ring of slots; Bulyan keeps as many leading slabs resident as the budget allows and re-streams only its
 * selected rows for the other columns.  Budget: free device memory plus what the call already holds,
 * minus 1 GiB, capped by the environment variable AFL_HOST_DEVICE_BYTES (bytes, read on every call).
 * If two slots and the n x n tables do not fit, AFL_ERR_UNSUPPORTED (the message states the bytes needed).
 * Results depend only on the input, n, d, ld and slab_cols, never on the budget or the free memory. */
int afl_defend_host(const char* rule, const float* G_host, int n, int64_t d, int64_t ld,
                    int users_count, int corrupted_count, float* out_host, int* idx_out,
                    int64_t slab_cols);

/* The rest of the host-buffer surface.  Each call is blocking, runs on the current device, streams
 * column slabs within afl_defend_host's budget (same AFL_ERR_UNSUPPORTED "needs N bytes" error) and
 * rounds `slab_cols` the same way; results depend only on the input and slab_cols.
 *
 * afl_sqdist_host — defences.py:16-21  _krum_create_distances.  Writes the n x n float64 squared-
 * distance table of the host matrix into d2_out (device float64[n*n], caller-owned), summed slab by
 * slab in slab order: the table afl_defend_host("Krum", ...) builds from the same arguments, bit for
 * bit.  No client limit: past 4096 clients every slab runs the SIMT kernel (afl_sqdist_partial). */
int afl_sqdist_host(const float* G_host, int n, int64_t d, int64_t ld, double* d2_out, int64_t slab_cols);

/* afl_bulyan_host — defences.py:55-70  bulyan.  afl_defend_host("Bulyan", ...) is this call with
 * sel_host = NULL.  sel_host (host int[users_count - 2*corrupted_count], may be NULL) receives the
 * selection in selection order, also on AFL_ERR_NO_WINNER, where the failed rounds hold -1.
 * AFL_ERR_PRECONDITION unless users_count >= 4f+3; n <= 4096 clients. */
int afl_bulyan_host(const float* G_host, int n, int64_t d, int64_t ld, int users_count, int corrupted_count,
                    float* out_host, int* sel_host, int64_t slab_cols);

/* afl_alie_host — malicious.py:14-19,35  Attack.attack + DriftAttack._attack_grads on host gradients.
 * rows: f separate host vectors of d fp32 (the users' own arrays; no stacked matrix is needed).  Each
 * slab packs the f row segments into a device slot and runs afl_alie on it.  mu_out, sigma_out,
 * crafted_out: host fp32[d], each may be NULL, with afl_alie's contract (bcast_rows = NULL):
 * crafted_out == mu_out reproduces the reference's in-place aliasing.  The column sums run down the
 * rows in float64, so the outputs equal one afl_alie over the stacked matrix, bit for bit. */
int afl_alie_host(const float* const* rows, int f, int64_t d, double z, float* mu_out, float* sigma_out,
                  float* crafted_out, int64_t slab_cols);

/* ---- batched device calls: many same-shape problems, one launch per stage --------------------------
 * `batch` independent problems of n <= 128 clients (one Gram tile), problem b at G + b * batch_stride
 * ELEMENTS, each with the same n, d, ld, users_count and corrupted_count.  The batch is a grid dimension
 * of the same kernels the single calls run, so every problem's result is the single device call's on
 * that problem (bit for bit: distance table, Krum index, Bulyan selection and output, trimmed mean,
 * mean, ALIE statistics; the Gram kernels' split count is chosen for the whole batch, so pin it with the
 * environment variable AFL_GRAM_SPLITS when comparing distance tables).  Device pointers; the calls only
 * enqueue work.  The tensor-core Gram path needs a 16-byte aligned base, ld and batch_stride with
 * batch_stride >= n * ld; anything else runs the SIMT Gram kernel.  Limits, checked before any CUDA call:
 * n > 128 or batch > 65535 -> AFL_ERR_UNSUPPORTED; batch < 1, a NULL pointer, or (batch > 1) a
 * batch_stride smaller than one problem's span ((n - 1) * ld + d) -> AFL_ERR_BAD_ARG.
 *
 * afl_defend_batched — defences.py:73-75 defend[rule] per problem.  rule as afl_defend_host.
 *   "Krum"        defences.py:23-42:  idx_out (device int[batch]) receives each problem's index (or -1);
 *                 users_count >= 2f+1 else AFL_ERR_PRECONDITION.
 *   "Bulyan"      defences.py:55-70:  out (device fp32[batch][d]) and sel_out (device int[batch][theta],
 *                 theta = users_count - 2f, selection order; a round with no eligible user writes -1 from
 *                 that round on in that problem's row, the other problems are unaffected); users_count
 *                 >= 4f+3 else AFL_ERR_PRECONDITION, and users_count == n.
 *   "TrimmedMean" defences.py:44-52 and "NoDefense" defences.py:13-14:  out (device fp32[batch][d]).
 * workspace: afl_batched_workspace_bytes(rule, batch, n, d, dtype) bytes, 256-byte aligned (0 on bad
 * arguments); TrimmedMean and NoDefense use none.  For Krum and Bulyan it begins with the batch's
 * squared-distance tables (float64[batch][n][n], afl_sqdist_partial's table of each problem), which the
 * caller may read once the call's work has run. */
size_t afl_batched_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype);
int afl_defend_batched(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                       int64_t ld, int dtype, int users_count, int corrupted_count, float* out, int* idx_out,
                       int* sel_out, void* workspace, size_t workspace_bytes, void* stream);

/* afl_alie_batched — malicious.py:10-27,34-36 per problem: afl_alie on rows 0..f-1 of every problem.
 * mu_out, sigma_out, crafted_out: device fp32[batch][d] (each may be NULL; crafted_out == mu_out
 * reproduces the reference's aliasing).  bcast_rows (may be NULL): the crafted vector of problem b is
 * written into rows 0..f-1 of bcast_rows + b * bcast_batch_stride (pitch bcast_ld), server.py:82-83. */
int afl_alie_batched(const void* G_mal, int batch, int64_t batch_stride, int f, int64_t d, int64_t ld,
                     int dtype, double z, float* mu_out, float* sigma_out, float* crafted_out,
                     float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* stream);

/* ---- per-problem batched calls: the same batches with corrupted_count (and ALIE's z) per problem ----------
 * The reference's results come from grids over z (--num_std, main.py:109) and the malicious share (--mal-prop,
 * main.py:106, f = int(mal_prop * N), main.py:21) as well as the seed.  These calls run such a grid as one batch:
 * problem b's result is, bit for bit, the single device call's on G[b] with its own f_b (and z_b).  Every other
 * argument, limit and stride rule is the scalar batched call's.  corrupted_counts / f / z are HOST arrays of `batch`
 * values; the call validates them, builds one small table of per-problem kernel parameters (the values the single
 * call derives: Krum's take, Bulyan's f and theta, the trimmed mean's kept count and pivot constants, ALIE's f, (float)z
 * and whether it writes) and copies it to the start of the workspace with cudaMemcpyAsync on `stream`.  The arrays may
 * be reused once the call returns.  Because that copy reads pageable memory, these calls cannot be captured into a
 * CUDA graph.  Checked before any CUDA call: a NULL array or f_b < 0 (ALIE: also f_b > n) -> AFL_ERR_BAD_ARG; a
 * workspace that is too small or not 256-byte aligned -> AFL_ERR_WORKSPACE; Krum's users_count >= 2f_b+1 and
 * Bulyan's users_count >= 4f_b+3 for every b, else AFL_ERR_PRECONDITION naming the first failing problem.
 *
 * afl_batched_each_workspace_bytes(rule, ...) — rule as afl_defend_batched, or "ALIE"; 0 on bad arguments, otherwise
 * at least afl_batched_workspace_bytes.  The parameter table comes first; for Krum and Bulyan the scalar call's layout
 * follows it, so that the squared-distance tables start at byte T = afl_batched_each_workspace_bytes -
 * afl_batched_workspace_bytes (the same tables the scalar call leaves at byte 0).
 *
 * afl_defend_batched_each — defences.py:73-75 defend[rule] per problem with f_b = corrupted_counts[b]:
 *   "Krum"        defences.py:23-42, take_b = len(sorted(...)[:users_count - f_b]).
 *   "TrimmedMean" defences.py:44-52, keep_b from n - f_b - 1 with Python slice semantics.
 *   "NoDefense"   defences.py:13-14, f_b is ignored as in the reference (no table, no workspace).
 *   "Bulyan"      defences.py:55-70, theta_b = users_count - 2f_b rounds, then the trimmed mean of those rows with
 *                 2f_b.  sel_out is device int[batch][theta_max], theta_max = users_count - 2 * min_b f_b: problem b
 *                 fills positions 0..theta_b-1 (-1 from a failed round on, as afl_defend_batched) and positions
 *                 theta_b..theta_max-1 with -2 ("no such round"). */
size_t afl_batched_each_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype);
int afl_defend_batched_each(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                            int64_t ld, int dtype, int users_count, const int* corrupted_counts, float* out,
                            int* idx_out, int* sel_out, void* workspace, size_t workspace_bytes, void* stream);

/* afl_alie_batched_each — malicious.py:10-27,34-36 per problem (DriftAttack(z_b).attack_rows(G[b], f_b)): problems
 * of n rows, of which rows 0..f_b-1 are malicious, f_b <= n.  Outputs and bcast_rows as afl_alie_batched.
 * f_b = 0 reads and writes no row and that problem's mu, sigma and crafted are NaN (the reference returns before
 * computing anything, malicious.py:11-12); z_b = 0 computes the statistics, crafted = mu - 0 * sigma, and writes no
 * row (malicious.py:20-21). */
int afl_alie_batched_each(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                          const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                          float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---- ragged batches: a different number of clients per problem ---------------------------------------------------
 * The reference's client count is a run parameter (--users-count, main.py:118), and Server.defend aggregates however many
 * users reported (server.py:87: defend[rule](users_grads, len(self.users), corrupted_count)).  These calls run problems of
 * different client counts, or rounds with partial participation, as one batch.  G is laid out as for
 * afl_defend_batched_each, n <= 128 rows per problem slot; problem b is its first rows[b] rows (1 <= rows[b] <= n).  Rows
 * rows[b]..n-1 of a slot are padding with any contents (NaN and +-inf included): no result depends on them.  rows,
 * users_counts and corrupted_counts are HOST arrays of `batch` values; problem b's result is the single device call's on
 * the rows[b] x d matrix G[b][:rows[b]] with users_counts[b] and corrupted_counts[b], bit for bit when both run the same
 * Gram operand format and split count (the format is chosen once for the batch from n, d and the dtype, as for a single
 * call of n clients; pin AFL_GRAM_SPLITS, and for fp32 AFL_GRAM_TF32X2, when comparing).  Checked before any CUDA call,
 * with the first failing problem named: a NULL array, rows[b] outside [1, n] or corrupted_counts[b] < 0 ->
 * AFL_ERR_BAD_ARG; the reference's asserts per problem -> AFL_ERR_PRECONDITION; a workspace that is too small or not
 * 256-byte aligned -> AFL_ERR_WORKSPACE.  Every other argument, limit and stride rule is afl_defend_batched_each's.
 *
 * afl_batched_rows_workspace_bytes(rule, ...) — rule as afl_defend_batched (0 otherwise, and on bad arguments); the same
 * bytes and layout as afl_batched_each_workspace_bytes (the parameter table, then for Krum and Bulyan the batch's n x n
 * squared-distance tables, whose entries between participating rows are the problems' own).
 *
 * afl_defend_batched_rows — defences.py:73-75 defend[rule](G[b][:rows[b]], users_counts[b], corrupted_counts[b]):
 *   "Krum"        defences.py:23-42 on rows[b] users (replaces the Python loop over server.py:87 for each client count):
 *                 idx_out[b] in [0, rows[b]) or -1 (rows[b] = 1, or no eligible user; the reference then returns
 *                 users_grads[-1], row rows[b] - 1).  users_counts[b] >= 2 corrupted_counts[b] + 1.
 *   "TrimmedMean" defences.py:44-52 over rows[b] rows (users_counts[b] is not used, as in the reference).
 *   "NoDefense"   defences.py:13-14, the mean of rows[b] rows (afl_mean's arithmetic).
 *   "Bulyan"      defences.py:55-70 with users_counts[b] >= 4 corrupted_counts[b] + 3 and users_counts[b] == rows[b]
 *                 (else AFL_ERR_UNSUPPORTED).  sel_out is device int[batch][theta_max], theta_max = max_b(users_counts[b]
 *                 - 2 corrupted_counts[b]); positions past problem b's theta_b hold -2, as afl_defend_batched_each. */
size_t afl_batched_rows_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype);
int afl_defend_batched_rows(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                            int64_t ld, int dtype, const int* rows, const int* users_counts, const int* corrupted_counts,
                            float* out, int* idx_out, int* sel_out, void* workspace, size_t workspace_bytes,
                            void* stream);

/* ---- large batches: up to 1024 clients per problem ----------------------------------------------------------------
 * The reference's larger runs have N = 500 and N = 1000 users (f = 240 at N = 1000).  These calls take the batches of
 * the calls above with 1 <= n <= 1024 rows per problem slot; n > 1024 -> AFL_ERR_UNSUPPORTED ("n <= 1024").
 *
 * afl_batched_large_workspace_bytes(rule, ...) — rule as afl_defend_batched; 0 on bad arguments and for n > 1024.  For
 * n <= 128 exactly afl_batched_rows_workspace_bytes.  For n > 128 the parameter table is followed by `batch` ints (the
 * problems grouped by trimmed-mean size class), then the layout of afl_batched_rows_workspace_bytes.
 *
 * afl_defend_batched_large — afl_defend_batched_rows with 1 <= n <= 1024: the same semantics, error codes, per-problem
 * error messages and output layouts (sel_out [batch][theta_max], -2 past theta_b).  rows may be NULL: n rows in every
 * problem.  rows, users_counts and corrupted_counts are HOST arrays.  Problem b's result is the single device call's
 * on G[b][:rows[b]] bit for bit when both run the same Gram operand format and split count (the format is chosen from
 * n, d and the dtype; for fp32 a single call at rows[b] > 128 runs the format a slot of n > 128 rows runs).  The
 * trimmed mean (TrimmedMean, Bulyan's second stage) of every problem runs the kernel its own row count selects.
 *
 * afl_alie_batched_large — afl_alie_batched_each without the client limit: f_b <= n for any n (ALIE is a column pass,
 * as afl_backdoor_start_batched).  Workspace: afl_batched_each_workspace_bytes("ALIE", batch, 1, d, dtype). */
size_t afl_batched_large_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype);
int afl_defend_batched_large(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                             int64_t ld, int dtype, const int* rows, const int* users_counts,
                             const int* corrupted_counts, float* out, int* idx_out, int* sel_out, void* workspace,
                             size_t workspace_bytes, void* stream);
int afl_alie_batched_large(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                           const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                           float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- attack-success metrics of a batch (SURVEY 8d "Attack-success (C5)") --------------------------------------
 * The reference logs test accuracy only (main.py:73-82); what a z x malicious-share sweep reports follows from its
 * conventions.  The malicious users are ids 0..f-1 (main.py:28), so in problem b rows f_b..n-1 are honest:
 *   h_b     = mean of rows f_b..n-1, afl_mean's arithmetic on that row range (bit for bit afl_mean of G[b] + f_b * ld);
 *   a_b     = the aggregate: agg + b * d (device fp32[batch][d], the output of Bulyan, TrimmedMean or NoDefense), or,
 *             with idx (device int[batch], Krum's idx_out) instead, row idx[b] of problem b upcast to fp32, read in
 *             place.  At most one of agg / idx; neither: selection statistics (and honest_out) only;
 *   dev_out   (device fp32[batch])      ||a_b - h_b|| / ||h_b||, both sums of squares accumulated in float64;
 *   sums_out  (device double[batch][2]) those two sums, (sum (a-h)^2, sum h^2): they ADD across column shards, and
 *             dev = sqrt(sums[0] / sums[1]) after the all-reduce;
 *   honest_out (device fp32[batch][d])  h_b;
 *   krum_hit  (device int[batch], needs idx)  1 when 0 <= idx[b] < f_b, else 0;
 *   mal_count, sel_count (device int[batch], need sel = device int[batch][sel_ld], Bulyan's sel_out): the entries of
 *             row b in [0, f_b), and the entries >= 0 (-1 = failed round, -2 = no such round are not counted).  The
 *             malicious fraction of the selection is mal_count / max(1, sel_count).
 * Every output may be NULL.  f_b >= n (no honest row) and idx[b] outside [0, n) (Krum found no eligible user: -1) read
 * no row and give NaN in dev_out and in the first sum of sums_out (f_b >= n: in both sums and in honest_out too).  A
 * zero or non-finite h gives what IEEE division gives (inf or NaN).  The sums are taken per tile of 1024 (fp32) or 2048 (bf16, fp16) columns and added in
 * a fixed order without atomics, so a result depends on the values, d and the dtype only: not on the pitch, the
 * alignment, the batch size or the device.
 * Device pointers; the calls only enqueue work.  There is no client limit (no distance table is built); batch <=
 * 65535 and the stride rule are afl_defend_batched's; batch = 1 with a plain [n][d] matrix is the single-problem
 * call.  Checked before any CUDA call: a NULL G, batch < 1, a short batch_stride, both agg and idx, an output
 * without its input, corrupted_count < 0 -> AFL_ERR_BAD_ARG; a dtype code other than afl_dtype's ->
 * AFL_ERR_UNSUPPORTED; a workspace smaller than afl_metrics_workspace_bytes(batch, n, d, dtype) (0 on bad arguments)
 * or not 256-byte aligned -> AFL_ERR_WORKSPACE (the scalar call needs none for selection statistics alone).
 * afl_attack_metrics_batched_each takes f_b = corrupted_counts[b], a HOST array of `batch` values copied to the start
 * of the workspace as the other *_each calls do (a NULL array or f_b < 0 -> AFL_ERR_BAD_ARG). */
size_t afl_metrics_workspace_bytes(int batch, int n, int64_t d, int dtype);
int afl_attack_metrics_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                               int corrupted_count, const float* agg, const int* idx, const int* sel, int sel_ld,
                               float* dev_out, double* sums_out, float* honest_out, int* krum_hit, int* mal_count,
                               int* sel_count, void* workspace, size_t workspace_bytes, void* stream);
int afl_attack_metrics_batched_each(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                    int dtype, const int* corrupted_counts, const float* agg, const int* idx,
                                    const int* sel, int sel_ld, float* dev_out, double* sums_out, float* honest_out,
                                    int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                    size_t workspace_bytes, void* stream);
/* afl_attack_metrics_batched_rows — afl_attack_metrics_batched_each on a ragged batch: problem b is its first rows[b]
 * rows (a HOST array, 1 <= rows[b] <= n, else AFL_ERR_BAD_ARG; NULL -> AFL_ERR_BAD_ARG), so its honest rows are
 * f_b..rows[b]-1 and h_b is afl_mean of those rows bit for bit; f_b >= rows[b] and idx[b] outside [0, rows[b]) give NaN
 * as above.  Rows past rows[b] are never read.  Same workspace as afl_attack_metrics_batched_each. */
int afl_attack_metrics_batched_rows(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                    int dtype, const int* rows, const int* corrupted_counts, const float* agg,
                                    const int* idx, const int* sel, int sel_ld, float* dev_out, double* sums_out,
                                    float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                    size_t workspace_bytes, void* stream);

/* ---- backdoor attack of a batch (backdoor.py:52-63, BackdoorAttack._attack_grads driven by malicious.py:10-27) -----
 * The crafting calls the attacker's model training (backdoor.py:56) in the middle, so it is two calls with the
 * caller's training between them.  Per problem b, with f_b = f[b], z_b = (float)z[b], lr_b = (float)lr[b] (HOST arrays
 * of `batch` values, copied into a parameter table at the start of the workspace as the other per-problem calls do):
 *   mu, sigma = afl_alie's statistics of rows 0..f_b-1 of G + b * batch_stride     malicious.py:17-18
 *   step      = mu * lr_b;  initial = w_b - step                                      backdoor.py:54
 *   mal       = the caller's training started from initial                          backdoor.py:56
 *   new_g     = (initial - (mal + step)) / lr_b  (IEEE division)                     backdoor.py:59-60
 *   crafted   = np.clip(new_g, mu - z_b*sigma, mu + z_b*sigma)  (NaN rules of afl_alie_band)   backdoor.py:62-63
 * and crafted is written over rows 0..f_b-1 (server.py:82-83), every operation one fp32 rounding as in the reference.
 * f_b = 0: NaN mu, sigma and crafted, no row read or written (malicious.py:11-12); z_b = 0: the statistics only,
 * crafted = mu, no row written (malicious.py:20-21).  Negative z_b and lr_b = 0 get what NumPy gives.
 *
 * afl_backdoor_start_batched — problems of n rows (no client limit: the pass is column-wise), f_b <= n, dtype fp32,
 * bf16 or fp16, batch_stride and batch <= 65535 as afl_defend_batched.  w: device fp32 params at w + b * w_batch_stride
 * (0: one [d] vector for every problem, else >= d).  Writes mu_out, sigma_out (afl_alie_batched_each's, bit for bit) and
 * initial_out, each device fp32[batch][d].
 * afl_backdoor_finish_batched — mu, sigma, initial as the start call left them; mal: device fp32 trained parameters at
 * mal + b * mal_batch_stride (>= d when batch > 1; read only for problems with f_b > 0 and z_b != 0).  Writes
 * crafted_out (device fp32[batch][d]) and, when bcast_rows is given (an fp32 matrix: a 16-bit one is written by the
 * caller), rows 0..f_b-1 of bcast_rows + b * bcast_batch_stride (pitch bcast_ld) of those problems.
 * Workspace of both: the table alone, afl_batched_each_workspace_bytes("ALIE", batch, 1, d, dtype) bytes (its size
 * depends on batch only, so any n <= 128 gives it), 256-byte aligned.  Device pointers; the calls only enqueue work.  Checked before any CUDA call: a NULL pointer
 * (outputs included; bcast_rows may be NULL), d < 1, batch < 1, f_b < 0 (start: f_b > n), a short batch_stride,
 * w_batch_stride, mal_batch_stride, bcast_ld or bcast_batch_stride -> AFL_ERR_BAD_ARG; batch > 65535 or another dtype
 * code -> AFL_ERR_UNSUPPORTED; a short or misaligned workspace -> AFL_ERR_WORKSPACE. */
int afl_backdoor_start_batched(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                               const int* f, const double* z, const double* lr, const float* w, int64_t w_batch_stride,
                               float* mu_out, float* sigma_out, float* initial_out, void* workspace,
                               size_t workspace_bytes, void* stream);
int afl_backdoor_finish_batched(int batch, int64_t d, const int* f, const double* z, const double* lr, const float* mu,
                                const float* sigma, const float* initial, const float* mal, int64_t mal_batch_stride,
                                float* crafted_out, float* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld,
                                void* workspace, size_t workspace_bytes, void* stream);

/* ---- device-parameter batched calls: per-problem arrays in device memory, capturable into a CUDA graph ---------
 * The per-problem calls above take their arrays on the host and build the parameter table there.  These take
 * rows, users_counts and corrupted_counts as DEVICE int32 arrays of `batch` values and z as a DEVICE float64 array,
 * build the table on the device (the host calls' row, field for field) and run the same kernels on it, so a result
 * is the host-parameter call's on the same values, bit for bit.  After the host checks below no call copies,
 * synchronises or allocates: every call only enqueues work and can be captured into a CUDA graph, whose replays read
 * whatever the arrays hold at that time.
 *
 * Per-problem checks run on the device, in the host calls' order: corrupted_counts[b] < 0 (or above the host
 * call's cap) or rows[b] outside [1, n] -> AFL_ERR_BAD_ARG; the reference's asserts (users_count >= 2f + 1 for Krum,
 * >= 4f + 3 for Bulyan) -> AFL_ERR_PRECONDITION; Bulyan's users_counts[b] != rows[b] -> AFL_ERR_UNSUPPORTED; and, after
 * Bulyan's selection, a failed round (sel_out[b][theta_b - 1] < 0) -> AFL_ERR_NO_WINNER.  The first code of problem b
 * is written to status[b] (DEVICE int32[batch], the caller's, left alone once nonzero: clear it to start again).  A
 * flagged problem runs with rows_b = n, users_count_b = n and f_b = 0 instead, which keeps every kernel inside its
 * slot; its outputs are then not the reference's, and only status says so.  The other problems are unaffected.
 *
 * Arguments follow the host calls: rows == NULL means n rows in every problem; users_counts == NULL means the scalar
 * users_count without rows, or rows with them.  Checked on the host before any CUDA call: NULL pointers, batch, the
 * stride rule, dtype and the workspace exactly as the host-parameter calls (status and corrupted_counts NULL ->
 * AFL_ERR_BAD_ARG).
 *
 * afl_batched_table_dev — writes only the table (ProblemParams[batch], 40 bytes a row, at the workspace start) and
 * status for rule "Krum", "Bulyan", "TrimmedMean", "NoDefense", "ALIE" (z required, rows ignored) or "AttackMetrics".
 * Workspace: afl_batched_each_workspace_bytes("ALIE", batch, 1, 1, 0) bytes or more.
 *
 * afl_defend_batched_dev — afl_defend_batched_rows (rows != NULL) or afl_defend_batched_each (rows == NULL) with
 * device arrays, n <= 128 (larger n -> AFL_ERR_UNSUPPORTED; afl_defend_batched_large_dev takes up to 1024).
 * Bulyan's sel_out is [batch][sel_ld] with sel_ld >= n (else AFL_ERR_BAD_ARG): theta_b
 * entries, then -2.  Workspace and layout: afl_batched_rows_workspace_bytes(rule, ...).
 *
 * afl_alie_batched_dev — afl_alie_batched_each / _large with device arrays, any n, f_b <= n.  bcast_rows (may be NULL)
 * has G's dtype: a bf16 or fp16 matrix is written in the kernel, rounded to nearest even (what torch's .to(dtype)
 * gives).  bcast_batch_stride >= (n - 1) * bcast_ld + d when batch > 1.  Workspace:
 * afl_batched_each_workspace_bytes("ALIE", batch, 1, d, dtype).
 *
 * afl_attack_metrics_batched_dev — afl_attack_metrics_batched_rows (rows != NULL) or _each with device arrays, any n.
 * Workspace: afl_metrics_workspace_bytes.
 *
 * afl_defend_batched_large_dev — afl_defend_batched_large with device arrays: the arguments of afl_defend_batched_dev
 * and 1 <= n <= 1024 (larger n -> AFL_ERR_UNSUPPORTED).  For n <= 128 it is afl_defend_batched_dev.  Above, the
 * per-problem checks, codes and safe row are afl_defend_batched_dev's, and the problems are grouped by trimmed-mean slot
 * class on the device, so the call still makes no host copy, synchronisation or allocation after its host checks.
 * Workspace: afl_batched_large_dev_workspace_bytes(rule, ...) — 0 on bad arguments and for n > 1024; for n <= 128
 * afl_batched_rows_workspace_bytes; above, afl_batched_large_workspace_bytes plus one 256-byte block at the end that
 * holds the class offsets, so every offset of the large call's layout (the table, perm, d2, dist, the Gram workspace
 * and the selection scratch) holds for this call too. */
int afl_batched_table_dev(const char* rule, int batch, int n, const int* rows, int users_count, const int* users_counts,
                          const int* corrupted_counts, const double* z, void* workspace, size_t workspace_bytes,
                          int* status, void* stream);
int afl_defend_batched_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                           int dtype, const int* rows, int users_count, const int* users_counts,
                           const int* corrupted_counts, float* out, int* idx_out, int* sel_out, int sel_ld,
                           void* workspace, size_t workspace_bytes, int* status, void* stream);
int afl_alie_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, int dtype,
                         const int* f, const double* z, float* mu_out, float* sigma_out, float* crafted_out,
                         void* bcast_rows, int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                         size_t workspace_bytes, int* status, void* stream);
size_t afl_batched_large_dev_workspace_bytes(const char* rule, int batch, int n, int64_t d, int dtype);
int afl_defend_batched_large_dev(const char* rule, const void* G, int batch, int64_t batch_stride, int n, int64_t d,
                                 int64_t ld, int dtype, const int* rows, int users_count, const int* users_counts,
                                 const int* corrupted_counts, float* out, int* idx_out, int* sel_out, int sel_ld,
                                 void* workspace, size_t workspace_bytes, int* status, void* stream);
int afl_attack_metrics_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                   int dtype, const int* rows, const int* corrupted_counts, const float* agg,
                                   const int* idx, const int* sel, int sel_ld, float* dev_out, double* sums_out,
                                   float* honest_out, int* krum_hit, int* mal_count, int* sel_count, void* workspace,
                                   size_t workspace_bytes, int* status, void* stream);

/* afl_attack_trace_dev — one round's attack figures of an fp32 batch, written into row *slot of caller-held tables, so
 * that a captured round replayed with an advancing slot (a training sweep's epoch counter) records every round.  The
 * device-parameter arguments (G .. ld, rows, corrupted_counts, workspace, status) are afl_attack_metrics_batched_dev's,
 * and the per-problem table and its status flags are that call's.  agg (fp32 [batch][d], required): the aggregate the
 * round applied; Krum's is the gathered winning row, so index -1 is measured as the row applied.  idx (int32 [batch],
 * may be NULL): Krum's index.  sel (int32 [batch][sel_ld], may be NULL): Bulyan's selection.  slot: a DEVICE int32.
 * Each output (may be NULL) is a table of n_slots rows at pitch table_ld >= batch; problem b writes entry
 * [*slot][b]:
 *   agg_dev   (fp32)  ||agg_b - h_b|| / ||h_b||, h_b the mean of the honest rows f_b .. rows_b - 1: the dev_out
 *                     afl_attack_metrics_batched_dev(agg = agg) gives, bit for bit;
 *   mal_dev   (fp32)  ||G[b, 0] - h_b|| / ||h_b|| when f_b > 0 (that call's dev_out with idx = 0, bit for bit), NaN
 *                     when f_b = 0;
 *   idx_out   (int32) idx[b] as given, -1 included (needs idx);
 *   mal_count, sel_count (int32)  that call's counts over row b of sel (need sel).
 * A slot outside [0, n_slots) writes nothing.  One column pass over the honest rows, agg and row 0, then one CTA per
 * problem; no host copy, synchronisation or allocation after the host checks, so the call can be captured.  Host
 * checks: NULL G, agg, slot, corrupted_counts or status, n_slots < 1, table_ld < batch, sel_ld < 1 with sel, a count
 * without sel, idx_out without idx and a short batch_stride -> AFL_ERR_BAD_ARG; a short or misaligned workspace ->
 * AFL_ERR_WORKSPACE.  Workspace: afl_attack_trace_workspace_bytes(batch, d) bytes, 256-byte aligned (0 on bad
 * arguments). */
size_t afl_attack_trace_workspace_bytes(int batch, int64_t d);
int afl_attack_trace_dev(const float* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, const int* rows,
                         const int* corrupted_counts, const float* agg, const int* idx, const int* sel, int sel_ld,
                         const int* slot, int n_slots, int64_t table_ld, float* agg_dev, float* mal_dev, int* idx_out,
                         int* mal_count, int* sel_count, void* workspace, size_t workspace_bytes, int* status,
                         void* stream);

/* ---- device-parameter backdoor crafting: afl_backdoor_start_batched / _finish_batched with f (int32), z and lr
 * (float64) as DEVICE arrays of `batch` values and a status array, as the other _dev calls take them.  The table is
 * built on the device, the host calls' row field for field, so on the same values each result equals the host call's
 * bit for bit.  n is the rows of a problem slot and bounds every f_b: f_b < 0 or f_b > n flags the problem with
 * AFL_ERR_BAD_ARG in status[b] and runs it with f_b = 0 (NaN mu, sigma and crafted; no row read or written).  For the
 * finish call n also bounds the rows bcast_rows receives: bcast_batch_stride >= (n - 1) * bcast_ld + d when batch > 1.
 * Workspace: afl_batched_each_workspace_bytes("ALIE", batch, 1, d, dtype) bytes, 256-byte aligned.  Every host check
 * is the host call's, plus status and f non-NULL; after them no call copies, synchronises or allocates. */
int afl_backdoor_start_batched_dev(const void* G, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld,
                                   int dtype, const int* f, const double* z, const double* lr, const float* w,
                                   int64_t w_batch_stride, float* mu_out, float* sigma_out, float* initial_out,
                                   void* workspace, size_t workspace_bytes, int* status, void* stream);
int afl_backdoor_finish_batched_dev(int batch, int n, int64_t d, const int* f, const double* z, const double* lr,
                                    const float* mu, const float* sigma, const float* initial, const float* mal,
                                    int64_t mal_batch_stride, float* crafted_out, float* bcast_rows,
                                    int64_t bcast_batch_stride, int64_t bcast_ld, void* workspace,
                                    size_t workspace_bytes, int* status, void* stream);

/* ---- MnistNet client gradients and evaluation (csrc/client_grad.cu): the training half of a sweep epoch ----------
 * The model is the harness's MnistNet (data_sets.py:13-24), log_softmax(fc2(relu(fc1(x)))), its d = 79,510 parameters
 * in ParamLayout order (fc1.weight [100][784], fc1.bias, fc2.weight [10][100], fc2.bias).  weights: device fp32
 * [batch][d], problem b's model.  x: device fp32 [n_sets][set_size][784] and y: device int64 [n_sets][set_size], one
 * data set per seed; data_index (device int32 [batch]) picks problem b's set (outside [0, n_sets): the problem is
 * skipped).  fp32 FFMA throughout, no atomics and every sum in a fixed order, so each result depends only on its
 * problem's weights, rows and m, never on batch, n or the other problems.  The calls only enqueue work on `stream`
 * (no allocation, copy or synchronisation), so they can be captured in a CUDA graph.  Checked before any CUDA call: a
 * NULL pointer, batch / n_sets / set size / m < 1 -> AFL_ERR_BAD_ARG; d != 79,510, m > 128 or batch > 65535 ->
 * AFL_ERR_UNSUPPORTED.
 *
 * afl_mnist_client_grads — user.py:76-92 for every client of every problem: client u < n_b = min(rows[b], n) (rows:
 * device int32 [batch]) computes the gradient of NLLLoss(mean) on its minibatch at problem b's weights and writes it
 * to columns [0, d) of row u of problem b, G + b * batch_stride + u * ld (fp32).  Nothing else of G is written.  Client
 * u's shard is training rows u, u + n_b, u + 2 n_b, ... (L = ceil((n_train - u) / n_b) of them); at epoch e = *epoch
 * (device int32, read when the kernel runs) it takes shard positions [k m, min(k m + m, L)), k = e mod ceil(L / m):
 * harness.Client.step's cycling position.  1 <= n <= 1024 clients and n <= n_train, else AFL_ERR_BAD_ARG /
 * AFL_ERR_UNSUPPORTED; ld >= d and (batch > 1) batch_stride >= (n - 1) * ld + d, else AFL_ERR_BAD_ARG.
 *
 * afl_mnist_client_grads_sets — afl_mnist_client_grads over training sets of their own lengths: set s starts at row
 * s * n_rows of x and y and its first set_len[s] rows are its training set (set_len: device int32 [n_sets], read when
 * the kernel runs), so client u of problem b takes rows u, u + n_b, ... of set data_index[b] with n_train =
 * set_len[data_index[b]].  A problem whose set length lies outside [n_b, n_rows] is skipped: none of its rows is
 * written.  The host checks are afl_mnist_client_grads' with n_rows for n_train, and a NULL set_len -> AFL_ERR_BAD_ARG.
 * With every set_len[s] = n_rows the results equal afl_mnist_client_grads(..., n_train = n_rows, ...) bit for bit.
 *
 * afl_mnist_evaluate — server.py:92-112 / harness.main's test loop for every problem: test batches of m rows (the last
 * one shorter), each batch's mean NLL in fp32, summed over the batches in order in float64 into
 * loss_sum[slot][b] (divide by n_test for the reported loss), and correct[slot][b] = the number of rows whose argmax
 * (torch's max(1) of the log-probabilities: the first NaN, else the first maximum) is the label.  slot = *slot_index
 * (device int32, read when the kernel runs); a slot outside [0, n_slots) writes nothing.  loss_sum: device float64
 * [n_slots][batch], correct: device int32 [n_slots][batch].  Workspace: afl_mnist_evaluate_workspace_bytes(batch, n_test, m) bytes, 256-byte aligned (else
 * AFL_ERR_WORKSPACE); 0 on bad arguments.  More than 65535 test batches -> AFL_ERR_UNSUPPORTED.
 *
 * afl_mnist_client_grads_each — afl_mnist_client_grads_sets with a minibatch size per problem: m is device int32
 * [batch] (read when the kernel runs) and problem b uses m[b] where the _sets call uses its scalar m, so its rows equal
 * afl_mnist_client_grads_sets(..., m = m[b], ...) bit for bit, whatever the other problems' sizes.  A problem whose
 * m[b] lies outside [1, max_m] is skipped: none of its rows is written.  The host checks are the _sets call's with
 * max_m for m (1 <= max_m <= 128), and a NULL m -> AFL_ERR_BAD_ARG.
 *
 * afl_mnist_evaluate_each — afl_mnist_evaluate with a test batch size per problem: problem b's test set runs in batches
 * of m[b] rows (m: device int32 [batch], read when the kernel runs), so loss_sum[slot][b] and correct[slot][b] equal
 * afl_mnist_evaluate's at m = m[b] bit for bit.  1 <= min_m <= max_m <= 128 (else AFL_ERR_BAD_ARG / _UNSUPPORTED); a
 * problem whose m[b] lies outside [min_m, max_m] writes nothing.  Workspace: afl_mnist_evaluate_workspace_bytes(batch,
 * n_test, min_m) bytes, 256-byte aligned (else AFL_ERR_WORKSPACE). */
int afl_mnist_client_grads(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                           int n_train, const int* data_index, const int* rows, int n, int m, const int* epoch,
                           float* G, int64_t batch_stride, int64_t ld, void* stream);
int afl_mnist_client_grads_sets(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                int n, int m, const int* epoch, float* G, int64_t batch_stride, int64_t ld,
                                void* stream);
size_t afl_mnist_evaluate_workspace_bytes(int batch, int n_test, int m);
int afl_mnist_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                       int n_test, const int* data_index, int m, const int* slot_index, int n_slots, double* loss_sum,
                       int* correct, void* workspace, size_t workspace_bytes, void* stream);
int afl_mnist_client_grads_each(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                int n, const int* m, int max_m, const int* epoch, float* G, int64_t batch_stride,
                                int64_t ld, void* stream);
int afl_mnist_evaluate_each(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                            int n_test, const int* data_index, const int* m, int min_m, int max_m,
                            const int* slot_index, int n_slots, double* loss_sum, int* correct, void* workspace,
                            size_t workspace_bytes, void* stream);

/* ---- the backdoor attacker's MnistNet (csrc/backdoor_train.cu): the model half of a backdoor sweep epoch ----------
 * Backdoor sets: x device fp32 [n_sets][max_len][784], y device int64 [n_sets][max_len], set_len device int32 [n_sets]
 * (set s is its first set_len[s] rows); data_index (device int32 [batch]) picks problem b's set.  Minibatches and test
 * batches are m rows (the last one shorter), 1 <= m <= 200.  One CTA per problem, fp32 FFMA throughout, no atomics and
 * every sum in a fixed order, so a problem's result depends only on its own inputs, never on batch or the other
 * problems.  The calls take no workspace and only enqueue work (no allocation, copy or synchronisation), so they can
 * be captured in a CUDA graph.  Checked before any CUDA call: a NULL pointer, batch / n_sets / max_len / m < 1 ->
 * AFL_ERR_BAD_ARG; d != 79,510, m > 200 or batch > 65535 -> AFL_ERR_UNSUPPORTED.
 *
 * afl_mnist_backdoor_train — harness.BackdoorTrainer.train (backdoor.py:108-159) for every problem that attacks:
 * f[b] > 0, z[b] != 0 and status[b] == 0 (device arrays, read when the kernel runs; batched.backdoor_rows' condition).
 * From p = p0 = initial[b] (device fp32 [batch][d]): if every row of the set is classified correctly (the BEFORE test),
 * out[b] = initial[b] bit for bit; otherwise mal_epochs passes over the set, one SGD step per minibatch from a fresh
 * optimiser: p <- p - 0.1 (g + 1e-4 p), g the gradient of NLLLoss(mean) + alpha * sum over the four tensors of
 * MSELoss(p, p0) (the MSE term only when alpha > 0).  The trained vector goes to out[b] (device fp32 [batch][d], must
 * not overlap initial).  A NaN distance loss (alpha > 0) or a NaN loss before a step sets status[b] to
 * AFL_ERR_NAN_DIST_LOSS or AFL_ERR_NAN_LOSS and stops that problem (out[b] then holds the last step's parameters); a set
 * index outside [0, n_sets) or a set length outside [1, max_len] sets AFL_ERR_BAD_ARG.  Any other problem's out[b] is
 * neither read nor written.  mal_epochs < 0 or a NaN alpha -> AFL_ERR_BAD_ARG.
 *
 * afl_mnist_backdoor_train_each — afl_mnist_backdoor_train with alpha and mal_epochs per problem: alpha is device fp32
 * [batch] and mal_epochs device int32 [batch] (read when the kernel runs), and problem b trains at alpha[b] and
 * mal_epochs[b], so its out[b] and status[b] equal afl_mnist_backdoor_train(..., alpha = alpha[b], mal_epochs =
 * mal_epochs[b], ...) bit for bit, whatever the other problems' values.  The MSE term, and AFL_ERR_NAN_DIST_LOSS, apply
 * only to problems with alpha[b] > 0; mal_epochs[b] = 0 returns initial[b] after the BEFORE test.  An attacking problem
 * whose alpha[b] is NaN or whose mal_epochs[b] < 0 gets status[b] = AFL_ERR_BAD_ARG, and its out[b] is neither read
 * nor written.  The host checks are the scalar call's without the value checks, and a NULL alpha or mal_epochs ->
 * AFL_ERR_BAD_ARG.
 *
 * afl_mnist_backdoor_test — BackdoorTrainer.test (backdoor.py:67-102; main.py:91-95's 'POST') at weights[b] (device
 * fp32 [batch][d]) for every problem: loss_sum[slot][b] = the float64 sum of the batches' fp32 mean NLL (divide by the
 * set length for the reported loss) and correct[slot][b] = the rows whose argmax (torch's: the first NaN, else the
 * first maximum) is the label.  slot = *slot_index (device int32, read when the kernel runs); a slot outside
 * [0, n_slots), or a problem whose set index or length is out of range, writes nothing.  loss_sum: device float64
 * [n_slots][batch], correct: device int32 [n_slots][batch]; n_slots < 1 -> AFL_ERR_BAD_ARG. */
int afl_mnist_backdoor_train(const float* initial, float* out, int batch, int64_t d, const float* x, const int64_t* y,
                             int n_sets, int max_len, const int* set_len, const int* data_index, const int* f,
                             const double* z, int* status, double alpha, int mal_epochs, int m, void* stream);
int afl_mnist_backdoor_train_each(const float* initial, float* out, int batch, int64_t d, const float* x,
                                  const int64_t* y, int n_sets, int max_len, const int* set_len, const int* data_index,
                                  const int* f, const double* z, int* status, const float* alpha,
                                  const int* mal_epochs, int m, void* stream);
int afl_mnist_backdoor_test(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                            int max_len, const int* set_len, const int* data_index, int m, const int* slot_index,
                            int n_slots, double* loss_sum, int* correct, void* stream);

/* ---- Cifar10Net training sweeps (csrc/cifar_grad.cu): the model half of a CIFAR10 sweep epoch ----------------------
 * harness.Cifar10Net (data_sets.py:33-52): conv1 3->16 k3, relu, maxpool 3, conv2 16->64 k4, relu, maxpool 4, fc1
 * 64->384, relu, fc2 384->192, relu, fc3 192->10, log_softmax; parameters in ParamLayout order (user.py:17-28),
 * D = 117,706.  The arguments are the afl_mnist_* ones above; x is device fp32 [n_sets][n_rows][3072], the NCHW
 * [3, 32, 32] images flattened.  The pools use floor mode, so only each image's 23x23 top-left corner reaches the loss,
 * and only it is computed; on finite values everything else contributes exact zeros (DESIGN 2.9).  MaxPool follows
 * torch's max_pool2d (first maximum, a NaN takes the index, the gradient goes to that index alone).  Same rules as the
 * MnistNet entries: fp32 FFMA only, no atomics, every sum in a fixed order, so a client's gradient depends only on its
 * weights, its rows and m; no allocation, copy or synchronisation, so the calls can be captured in a CUDA graph.
 * Checked before any CUDA call: a NULL pointer, batch / n_sets / set size / m < 1 -> AFL_ERR_BAD_ARG; d != 117,706,
 * m > 128 or batch > 65535 -> AFL_ERR_UNSUPPORTED.
 *
 * afl_cifar10_client_grads — user.py:76-92 with Cifar10Net for every client of every problem: afl_mnist_client_grads'
 * clients, shards, minibatches (from *epoch) and limits on n, ld and batch_stride.  Only columns [0, d) of rows u <
 * min(rows[b], n) of each problem are written.  No workspace: the kernel accumulates the weight gradients in the row.
 *
 * afl_cifar10_client_grads_sets — afl_cifar10_client_grads over sets of their own lengths: afl_mnist_client_grads_sets'
 * pitch n_rows, device set_len, skip rule and checks.
 *
 * afl_cifar10_evaluate — server.py:92-112 / harness.main's test loop with Cifar10Net: afl_mnist_evaluate's batches,
 * float64 loss sums, correct counts by torch's argmax, NaN loss for a label outside 0..9, slot rule and workspace
 * (afl_cifar10_evaluate_workspace_bytes(batch, n_test, m) bytes, 256-byte aligned).
 *
 * afl_cifar10_client_grads_each, afl_cifar10_evaluate_each — the MnistNet _each calls with Cifar10Net: per-problem m
 * (device int32 [batch]), max_m (and min_m for the test), the skip rules and the workspace at min_m; each problem's
 * results equal the scalar call's at m = m[b] bit for bit. */
int afl_cifar10_client_grads(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                             int n_train, const int* data_index, const int* rows, int n, int m, const int* epoch,
                             float* G, int64_t batch_stride, int64_t ld, void* stream);
int afl_cifar10_client_grads_sets(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                  int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                  int n, int m, const int* epoch, float* G, int64_t batch_stride, int64_t ld,
                                  void* stream);
size_t afl_cifar10_evaluate_workspace_bytes(int batch, int n_test, int m);
int afl_cifar10_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                         int n_test, const int* data_index, int m, const int* slot_index, int n_slots,
                         double* loss_sum, int* correct, void* workspace, size_t workspace_bytes, void* stream);
int afl_cifar10_client_grads_each(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                  int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                  int n, const int* m, int max_m, const int* epoch, float* G, int64_t batch_stride,
                                  int64_t ld, void* stream);
int afl_cifar10_evaluate_each(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                              int n_sets, int n_test, const int* data_index, const int* m, int min_m, int max_m,
                              const int* slot_index, int n_slots, double* loss_sum, int* correct, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- the backdoor attacker's Cifar10Net (csrc/cifar_backdoor.cu): the model half of a CIFAR10 backdoor sweep epoch --
 * The afl_mnist_backdoor_* entries above with Cifar10Net (D = 117,706): the same backdoor sets, activity condition,
 * BEFORE test, SGD steps, status codes, slot rule and outputs, with x device fp32 [n_sets][max_len][3072] (the NCHW
 * [3, 32, 32] images flattened) and the MSE term over Cifar10Net's ten tensors.  The forward and backward passes are
 * afl_cifar10_client_grads' (the 23x23 corner, torch's max_pool2d rules), so one training step's NLL gradient is that
 * call's on the same rows bit for bit.  One CTA per problem for the training, fp32 FFMA throughout, no atomics and
 * every sum in a fixed order, so a problem's result depends only on its own inputs; no allocation, copy or
 * synchronisation, so the calls can be captured in a CUDA graph.  Checked before any CUDA call: a NULL pointer, batch /
 * n_sets / max_len / m < 1, mal_epochs < 0, a NaN alpha or a short workspace -> AFL_ERR_BAD_ARG; d != 117,706,
 * m > 200 or batch > 65535 -> AFL_ERR_UNSUPPORTED.
 *
 * afl_cifar10_backdoor_train — afl_mnist_backdoor_train's contract.  workspace: device memory of at least
 * afl_cifar10_backdoor_train_workspace_bytes(batch) bytes (4-byte aligned; problem b's step gradient lives in floats
 * [b d, b d + d)), overlapping neither initial nor out.
 *
 * afl_cifar10_backdoor_train_each — afl_mnist_backdoor_train_each's per-problem alpha (device fp32 [batch]) and
 * mal_epochs (device int32 [batch]) with afl_cifar10_backdoor_train's workspace: each problem equals the scalar call at
 * its own values bit for bit, and a NaN alpha[b] or a negative mal_epochs[b] sets status[b] = AFL_ERR_BAD_ARG before
 * out[b] is touched.  A NULL alpha or mal_epochs -> AFL_ERR_BAD_ARG.
 *
 * afl_cifar10_backdoor_test — afl_mnist_backdoor_test's contract, as one CTA per (test batch, problem) and a finish
 * kernel that sums the batches in order.  workspace: afl_cifar10_backdoor_test_workspace_bytes(batch, max_len, m)
 * bytes, 256-byte aligned; ceil(max_len / m) > 65535 -> AFL_ERR_UNSUPPORTED. */
size_t afl_cifar10_backdoor_train_workspace_bytes(int batch);
int afl_cifar10_backdoor_train(const float* initial, float* out, int batch, int64_t d, const float* x, const int64_t* y,
                               int n_sets, int max_len, const int* set_len, const int* data_index, const int* f,
                               const double* z, int* status, double alpha, int mal_epochs, int m, void* workspace,
                               size_t workspace_bytes, void* stream);
int afl_cifar10_backdoor_train_each(const float* initial, float* out, int batch, int64_t d, const float* x,
                                    const int64_t* y, int n_sets, int max_len, const int* set_len,
                                    const int* data_index, const int* f, const double* z, int* status,
                                    const float* alpha, const int* mal_epochs, int m, void* workspace,
                                    size_t workspace_bytes, void* stream);
size_t afl_cifar10_backdoor_test_workspace_bytes(int batch, int max_len, int m);
int afl_cifar10_backdoor_test(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                              int max_len, const int* set_len, const int* data_index, int m, const int* slot_index,
                              int n_slots, double* loss_sum, int* correct, void* workspace, size_t workspace_bytes,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AFL_B200_H_ */
