// Training-sweep code that does not depend on the net: the 10-class head, the client minibatch, the attacker's SGD
// step, and the host-side argument checks and evaluation workspace of the MnistNet (mnist_net.cuh) and Cifar10Net
// (cifar_net.cuh) calls (DESIGN 2.6).
#pragma once
#include "afl_common.cuh"

namespace afl {
namespace train {

constexpr int kClasses = 10;                         // both nets' output classes
constexpr float kLr = 0.1f, kWeightDecay = 1e-4f;   // backdoor.py:134

// A weight load.  kNc: through the read-only data cache (__ldg), for weights no thread writes while the kernel runs;
// otherwise an ordinary load, for the backdoor trainers' parameters, which the kernel updates in place between steps.
template <bool kNc>
__device__ __forceinline__ float ldw(const float* p) {
  if constexpr (kNc) return __ldg(p);
  else return *p;
}

// torch.relu: NaN stays NaN (fmaxf would turn it into 0).
__device__ __forceinline__ float relu(float v) { return v > 0.f || v != v ? v : 0.f; }

// torch's log_softmax of one row of logits: z - max - log(sum_c exp(z_c - max)), c in order.  The output is either all
// NaN (a NaN or infinite logit, or every logit -inf, makes the sum NaN) or free of NaN.
__device__ __forceinline__ void log_softmax_row(const float* zrow, float* logp) {
  float z[kClasses];
#pragma unroll
  for (int c = 0; c < kClasses; ++c) z[c] = zrow[c];
  float mx = z[0];
#pragma unroll
  for (int c = 1; c < kClasses; ++c) mx = fmaxf(mx, z[c]);
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < kClasses; ++c) sum += expf(z[c] - mx);
  const float lse = logf(sum);
#pragma unroll
  for (int c = 0; c < kClasses; ++c) logp[c] = z[c] - mx - lse;
}

// One row of logits z: returns its NLL (-logp[label]; NaN for a label outside 0..9) and sets *hit when torch's
// out.max(1)[1] is the label (the first NaN, else the first maximum).
__device__ __forceinline__ float row_head(const float* z, int yi, bool* hit) {
  float lp[kClasses];
  log_softmax_row(z, lp);
  int best = 0;
#pragma unroll
  for (int c = 1; c < kClasses; ++c)
    if (lp[best] == lp[best] && (lp[c] != lp[c] || lp[c] > lp[best])) best = c;
  *hit = best == yi;
  return yi >= 0 && yi < kClasses ? -lp[yi] : __int_as_float(0x7fc00000);
}

// NLLLoss(mean) of an mb-row minibatch through log_softmax's backward, for one row with log-probabilities lp and label
// yi: delta[c] = (softmax - onehot) / mb.  delta may be the row's logits.
__device__ __forceinline__ void row_delta(const float* lp, int yi, float fmb, float* delta) {
#pragma unroll
  for (int c = 0; c < kClasses; ++c) delta[c] = (expf(lp[c]) - (c == yi ? 1.f : 0.f)) / fmb;
}

// Client u's minibatch at epoch e (harness.Client.step's cycling position in closed form): its shard is rows u, u + n,
// u + 2n, ... of the training set, L = ceil((n_train - u) / n) long; at epoch e it takes shard positions
// [k m, min(k m + m, L)) with k = e mod ceil(L / m).  Returns the first position; *mb receives the row count.
__device__ __forceinline__ int batch_start(int n_train, int n, int u, int m, int e, int* mb) {
  const int L = (n_train - u + n - 1) / n;
  const int q = (L + m - 1) / m;
  int k = e % q;
  if (k < 0) k += q;
  const int lo = k * m;
  *mb = min(lo + m, L) - lo;
  return lo;
}

// Problem b's minibatch (or test batch) size: m, or m_each[b] for the per-problem (_each) calls, where a size outside
// [lo, m] returns 0 and the caller skips the problem.  The scalar calls pass m_each = nullptr.
__device__ __forceinline__ int problem_m(const int* m_each, int b, int lo, int m) {
  if (!m_each) return m;
  const int mb = m_each[b];
  return mb >= lo && mb <= m ? mb : 0;
}

// One SGD step of one element (backdoor.py:134-153 with torch.optim.SGD's first step of a fresh optimiser): g is the
// NLL gradient; with alpha > 0 the MSE term's ((p - p0) * 2/numel) * alpha is added (mse_loss's backward); then
// d_p = g + 1e-4 p and p - 0.1 d_p.  *bad is set when the new p - p0 is NaN, which makes the next dist loss NaN.
__device__ __forceinline__ float sgd(float p, float p0, float g, float norm, float alpha, bool dist, bool* bad) {
  if (dist) g = __fadd_rn(g, __fmul_rn(__fmul_rn(__fsub_rn(p, p0), norm), alpha));
  const float dp = __fmaf_rn(kWeightDecay, p, g);
  const float np = __fmaf_rn(-kLr, dp, p);
  const float r = __fsub_rn(np, p0);
  if (r != r) *bad = true;
  return np;
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

// The size checks every training call shares (pointers are checked by the callers).  `net` and `net_d` name the layout,
// `max_m` is the kernels' minibatch limit and `rows_name` the row-count argument as the message calls it.
inline int check_common(const char* who, const char* net, int64_t net_d, int max_m, const char* rows_name, int batch,
                        int64_t d, int n_sets, int n_rows, int m) {
  if (batch < 1 || n_sets < 1 || n_rows < 1 || m < 1) {
    set_error("%s: batch, n_sets, %s and m must be >= 1 (got %d, %d, %d, %d)", who, rows_name, batch, n_sets, n_rows,
              m);
    return AFL_ERR_BAD_ARG;
  }
  if (d != net_d) {
    set_error("%s: the %s layout has D = %lld parameters (got %lld)", who, net, static_cast<long long>(net_d),
              static_cast<long long>(d));
    return AFL_ERR_UNSUPPORTED;
  }
  if (m > max_m) { set_error("%s: batch size m <= %d (got %d)", who, max_m, m); return AFL_ERR_UNSUPPORTED; }
  if (batch > 65535) { set_error("%s: batch <= 65535 problems (got %d)", who, batch); return AFL_ERR_UNSUPPORTED; }
  return AFL_OK;
}

// The arguments of afl_*_client_grads[_sets]: n clients per problem, each writing D = net_d floats into its row of G.
inline int check_client_grads(const char* who, const char* net, int64_t net_d, int max_m, const float* weights,
                              int batch, int64_t d, const float* x, const int64_t* y, int n_sets, int n_rows,
                              const int* data_index, const int* rows, int n, int m, const int* epoch, const float* G,
                              int64_t batch_stride, int64_t ld) {
  if (!weights || !x || !y || !data_index || !rows || !epoch || !G) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = check_common(who, net, net_d, max_m, "the set size", batch, d, n_sets, n_rows, m)) return rc;
  if (n < 1 || n > 1024) { set_error("%s: 1 <= n <= 1024 clients per problem (got %d)", who, n); return n < 1 ? AFL_ERR_BAD_ARG : AFL_ERR_UNSUPPORTED; }
  if (n > n_rows) { set_error("%s: n (%d) exceeds the training set size (%d)", who, n, n_rows); return AFL_ERR_BAD_ARG; }
  if (ld < d || (batch > 1 && batch_stride < (n - 1) * ld + d)) {
    set_error("%s: ld (%lld) < d or batch_stride (%lld) makes problems overlap", who, static_cast<long long>(ld),
              static_cast<long long>(batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  return AFL_OK;
}

// The workspace of a batched test over sets of n_rows rows in m-row batches: every (problem, batch)'s fp32 mean NLL,
// then its correct count, each array 256-byte aligned.
struct EvalWorkspace {
  float* batch_loss;
  int* batch_correct;
  int nb;                 // batches per problem
};

inline int64_t eval_batches(int n_rows, int m) { return (int64_t(n_rows) + m - 1) / m; }

inline size_t eval_workspace_bytes(int batch, int n_rows, int m) {
  if (batch < 1 || n_rows < 1 || m < 1) return 0;
  const size_t per = static_cast<size_t>(batch) * eval_batches(n_rows, m);
  return align_up(per * sizeof(float), 256) + align_up(per * sizeof(int), 256);
}

// Checks the caller's workspace (a short or misaligned one returns short_rc) and the batch count, and carves it.
inline int carve_eval_workspace(const char* who, void* workspace, size_t workspace_bytes, int batch, int n_rows, int m,
                                int short_rc, EvalWorkspace* ws) {
  const size_t need = eval_workspace_bytes(batch, n_rows, m);
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 256) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, workspace_bytes, need);
    return short_rc;
  }
  const int64_t nb = eval_batches(n_rows, m);
  if (nb > 65535) { set_error("%s: at most 65535 test batches (got %lld)", who, static_cast<long long>(nb)); return AFL_ERR_UNSUPPORTED; }
  ws->batch_loss = static_cast<float*>(workspace);
  ws->batch_correct = reinterpret_cast<int*>(static_cast<char*>(workspace) +
                                             align_up(static_cast<size_t>(batch) * nb * sizeof(float), 256));
  ws->nb = static_cast<int>(nb);
  return AFL_OK;
}

// The arguments of afl_*_evaluate, then the workspace carve.
inline int check_evaluate(const char* who, const char* net, int64_t net_d, int max_m, const float* weights, int batch,
                          int64_t d, const float* x, const int64_t* y, int n_sets, int n_test, const int* data_index,
                          int m, const int* slot_index, int n_slots, const double* loss_sum, const int* correct,
                          void* workspace, size_t workspace_bytes, EvalWorkspace* ws) {
  if (!weights || !x || !y || !data_index || !slot_index || !loss_sum || !correct || !workspace) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = check_common(who, net, net_d, max_m, "the set size", batch, d, n_sets, n_test, m)) return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  return carve_eval_workspace(who, workspace, workspace_bytes, batch, n_test, m, AFL_ERR_WORKSPACE, ws);
}

// The arguments of afl_*_evaluate_each: afl_*_evaluate's with the per-problem sizes m (device int32 [batch]) in
// [min_m, max_m], and the workspace carved for the batch count at min_m.
inline int check_evaluate_each(const char* who, const char* net, int64_t net_d, int max_batch, const float* weights,
                               int batch, int64_t d, const float* x, const int64_t* y, int n_sets, int n_test,
                               const int* data_index, const int* m, int min_m, int max_m, const int* slot_index,
                               int n_slots, const double* loss_sum, const int* correct, void* workspace,
                               size_t workspace_bytes, EvalWorkspace* ws) {
  if (!m) { set_error("%s: a pointer argument is NULL", who); return AFL_ERR_BAD_ARG; }
  if (min_m > max_m) { set_error("%s: min_m (%d) > max_m (%d)", who, min_m, max_m); return AFL_ERR_BAD_ARG; }
  if (int rc = check_evaluate(who, net, net_d, max_batch, weights, batch, d, x, y, n_sets, n_test, data_index, max_m,
                              slot_index, n_slots, loss_sum, correct, workspace, workspace_bytes, ws))
    return rc;
  if (min_m < 1) { set_error("%s: min_m must be >= 1 (got %d)", who, min_m); return AFL_ERR_BAD_ARG; }
  return carve_eval_workspace(who, workspace, workspace_bytes, batch, n_test, min_m, AFL_ERR_WORKSPACE, ws);
}

// loss_sum[slot][b] = sum_t batch_loss[b][t] in float64, t in order (harness.main's `test_loss += ....item()`);
// correct[slot][b] = sum_t batch_correct[b][t], for every problem whose set index is in range: t < ws.nb, or with
// m_each t < ceil(n_test / m_each[b]) for a size in [min_m, max_m] (any other size writes nothing).  Defined in
// client_grad.cu.
int evaluate_finish(cudaStream_t stream, int batch, const EvalWorkspace& ws, const int* data_index, int n_sets,
                    const int* slot_index, int n_slots, double* loss_sum, int* correct, const int* m_each = nullptr,
                    int min_m = 0, int max_m = 0, int n_test = 0);

inline bool overlap(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return x < y + nb && y < x + na;
}

}  // namespace train
}  // namespace afl
