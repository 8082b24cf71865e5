// Batched MnistNet client gradients and test-set evaluation: the training half of a sweep epoch (sweep.py).
//
// The net is harness.MnistNet (data_sets.py:13-24): log_softmax(fc2(relu(fc1(x)))), fc1 [100, 784], fc2 [10, 100],
// flattened in ParamLayout order (fc1.weight, fc1.bias, fc2.weight, fc2.bias; D = 79,510).  One CTA runs one client
// (grid x = client, y = problem): it builds its minibatch's row list from the device epoch counter, runs the forward
// pass, the NLL(mean) backward and writes the gradient straight into its row of the client matrix.  Every sum is a
// sequential loop of one thread in a fixed order and nothing is atomic, so a client's gradient depends only on its
// weights, its rows and m.  Full fp32 FFMA throughout (the reference trains in fp32; no TF32).
#include "afl_common.cuh"

namespace afl {
namespace mnist {

constexpr int kIn = 784, kHid = 100, kOut = 10;
constexpr int64_t kD = int64_t(kHid) * kIn + kHid + kOut * kHid + kOut;        // 79,510
constexpr int kOffB1 = kHid * kIn, kOffW2 = kOffB1 + kHid, kOffB2 = kOffW2 + kOut * kHid;
constexpr int kThreads = 256;
constexpr int kMaxBatch = 128;          // minibatch rows a CTA holds (16 row groups of up to 8 rows)
constexpr int kHidPad = 112;            // forward: 16 column lanes x 7 hidden units
constexpr int kKc1 = 16;                // forward k-chunk (784 = 49 x 16)
constexpr int kLdX1 = kMaxBatch + 1;    // Xs[k][row]: the transposed store is conflict-free
constexpr int kLdW1 = kHidPad + 1;      // Ws[k][unit]
constexpr int kKc3 = 56;                // weight-gradient column chunk (784 = 14 x 56): 8 lanes x 7 columns
constexpr int kLdA = kHid + 1;          // A / delta1 rows

// shared memory, in floats
constexpr int kSmA = kMaxBatch * kLdA;                  // relu(fc1) rows, then delta1 rows
constexpr int kSmP = kMaxBatch * kOut;                  // logits, then delta2 rows
constexpr int kSmW2 = kOut * kHid;
constexpr int kSmFwd = kKc1 * kLdX1 + kKc1 * kLdW1;
constexpr int kSmX3 = kMaxBatch * kKc3;
constexpr int kSmScratch = kSmFwd > kSmX3 ? kSmFwd : kSmX3;
constexpr size_t kSmemBytes = sizeof(float) * (kSmA + kSmP + kSmW2 + kSmScratch) + sizeof(int) * 2 * kMaxBatch;

struct Smem {
  float* A; float* P; float* W2; float* scratch; int* row; int* label;
};

__device__ __forceinline__ Smem carve(float* base) {
  Smem s;
  s.A = base; s.P = s.A + kSmA; s.W2 = s.P + kSmP; s.scratch = s.W2 + kSmW2;
  s.row = reinterpret_cast<int*>(s.scratch + kSmScratch); s.label = s.row + kMaxBatch;
  return s;
}

// torch.relu: NaN stays NaN (fmaxf would turn it into 0).
__device__ __forceinline__ float relu(float v) { return v > 0.f || v != v ? v : 0.f; }

// Forward through relu(fc1): A[i][j] = relu(sum_k X[row_i][k] W1[j][k] + b1[j]) for i < mb, j < 100.  Thread (tx, ty)
// owns hidden units tx + 16c and rows ty + 16r; each of its sums runs k = 0..783 in order, then adds the bias.
template <int RT>
__device__ __forceinline__ void forward_hidden(const float* __restrict__ xs, const float* __restrict__ w, int mb,
                                               const Smem& s) {
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  float* Xs = s.scratch;
  float* Ws = s.scratch + kKc1 * kLdX1;
  float acc[RT][7];
#pragma unroll
  for (int r = 0; r < RT; ++r)
#pragma unroll
    for (int c = 0; c < 7; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < kIn; k0 += kKc1) {
    for (int idx = t; idx < 16 * RT * kKc1; idx += kThreads) {
      const int i = idx / kKc1, kk = idx % kKc1;
      Xs[kk * kLdX1 + i] = i < mb ? xs[int64_t(s.row[i]) * kIn + k0 + kk] : 0.f;
    }
    for (int idx = t; idx < kHidPad * kKc1; idx += kThreads) {
      const int j = idx / kKc1, kk = idx % kKc1;
      Ws[kk * kLdW1 + j] = j < kHid ? w[j * kIn + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kKc1; ++kk) {
      float xv[RT], wv[7];
#pragma unroll
      for (int r = 0; r < RT; ++r) xv[r] = Xs[kk * kLdX1 + ty + 16 * r];
#pragma unroll
      for (int c = 0; c < 7; ++c) wv[c] = Ws[kk * kLdW1 + tx + 16 * c];
#pragma unroll
      for (int r = 0; r < RT; ++r)
#pragma unroll
        for (int c = 0; c < 7; ++c) acc[r][c] = fmaf(xv[r], wv[c], acc[r][c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int c = 0; c < 7; ++c) {
    const int j = tx + 16 * c;
    if (j >= kHid) continue;
    const float bj = w[kOffB1 + j];
#pragma unroll
    for (int r = 0; r < RT; ++r) {
      const int i = ty + 16 * r;
      if (i < mb) s.A[i * kLdA + j] = relu(acc[r][c] + bj);
    }
  }
}

// logits P[i][c] = sum_j A[i][j] W2[c][j] (j in order) + b2[c]; W2 is staged into s.W2 first.
__device__ __forceinline__ void forward_logits(const float* __restrict__ w, int mb, const Smem& s) {
  for (int idx = threadIdx.x; idx < mb * kOut; idx += kThreads) {
    const int i = idx / kOut, c = idx % kOut;
    float z = 0.f;
    for (int j = 0; j < kHid; ++j) z = fmaf(s.A[i * kLdA + j], s.W2[c * kHid + j], z);
    s.P[i * kOut + c] = z + w[kOffB2 + c];
  }
}

// torch's log_softmax: z - max - log(sum_c exp(z_c - max)), c in order.
__device__ __forceinline__ void log_softmax_row(const float* z, float* logp) {
  float mx = z[0];
#pragma unroll
  for (int c = 1; c < kOut; ++c) mx = fmaxf(mx, z[c]);
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < kOut; ++c) sum += expf(z[c] - mx);
  const float lse = logf(sum);
#pragma unroll
  for (int c = 0; c < kOut; ++c) logp[c] = z[c] - mx - lse;
}

__device__ __forceinline__ void stage_w2(const float* __restrict__ w, const Smem& s) {
  for (int idx = threadIdx.x; idx < kOut * kHid; idx += kThreads) s.W2[idx] = w[kOffW2 + idx];
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

template <int RT>
__global__ void __launch_bounds__(kThreads, 2)
client_grad_kernel(const float* __restrict__ weights, const float* __restrict__ x, const int64_t* __restrict__ y,
                   int n_sets, int n_rows, const int* __restrict__ set_len, const int* __restrict__ data_index,
                   const int* __restrict__ rows, int n_max, int m, const int* __restrict__ epoch, float* __restrict__ G,
                   int64_t batch_stride, int64_t ld) {
  const int u = blockIdx.x, b = blockIdx.y;
  const int n = min(rows[b], n_max);
  const int set = data_index[b];
  if (u >= n || set < 0 || set >= n_sets) return;                 // block-uniform, before any barrier
  const int n_train = set_len ? set_len[set] : n_rows;            // no set_len: every set is n_rows long
  if (n_train < n || n_train > n_rows) return;
  extern __shared__ float smem[];
  const Smem s = carve(smem);
  const float* w = weights + int64_t(b) * kD;
  const float* xs = x + int64_t(set) * n_rows * kIn;
  const int64_t* ys = y + int64_t(set) * n_rows;
  int mb;
  const int lo = batch_start(n_train, n, u, m, *epoch, &mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    const int r = u + n * (lo + i);
    s.row[i] = r;
    s.label[i] = static_cast<int>(ys[r]);
  }
  stage_w2(w, s);
  __syncthreads();
  forward_hidden<RT>(xs, w, mb, s);
  __syncthreads();
  forward_logits(w, mb, s);
  __syncthreads();
  // delta2 = (softmax - onehot) / mb: NLLLoss(mean) through log_softmax's backward
  const float fmb = static_cast<float>(mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    float z[kOut], lp[kOut];
#pragma unroll
    for (int c = 0; c < kOut; ++c) z[c] = s.P[i * kOut + c];
    log_softmax_row(z, lp);
    const int yi = s.label[i];
#pragma unroll
    for (int c = 0; c < kOut; ++c) s.P[i * kOut + c] = (expf(lp[c]) - (c == yi ? 1.f : 0.f)) / fmb;
  }
  __syncthreads();
  float* g = G + int64_t(b) * batch_stride + int64_t(u) * ld;
  // fc2: dW2[c][j] = sum_i delta2[i][c] A[i][j], db2[c] = sum_i delta2[i][c] (i in order)
  for (int idx = threadIdx.x; idx < kOut * kHid + kOut; idx += kThreads) {
    float acc = 0.f;
    if (idx < kOut * kHid) {
      const int c = idx / kHid, j = idx % kHid;
      for (int i = 0; i < mb; ++i) acc = fmaf(s.P[i * kOut + c], s.A[i * kLdA + j], acc);
      g[kOffW2 + idx] = acc;
    } else {
      const int c = idx - kOut * kHid;
      for (int i = 0; i < mb; ++i) acc += s.P[i * kOut + c];
      g[kOffB2 + c] = acc;
    }
  }
  __syncthreads();
  // delta1 = delta2 W2 where A is not <= 0, in place of A (threshold_backward: zero where the ReLU output is <= 0, the
  // gradient elsewhere, a NaN output included)
  for (int idx = threadIdx.x; idx < mb * kHid; idx += kThreads) {
    const int i = idx / kHid, j = idx % kHid;
    float d = 0.f;
#pragma unroll
    for (int c = 0; c < kOut; ++c) d = fmaf(s.P[i * kOut + c], s.W2[c * kHid + j], d);
    s.A[i * kLdA + j] = s.A[i * kLdA + j] <= 0.f ? 0.f : d;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < kHid; j += kThreads) {
    float acc = 0.f;
    for (int i = 0; i < mb; ++i) acc += s.A[i * kLdA + j];
    g[kOffB1 + j] = acc;
  }
  // fc1: dW1[j][k] = sum_i delta1[i][j] X[row_i][k], 56 columns at a time.  Thread (tx, ty) owns columns tx + 8e and
  // units ty + 32c; warps 1..7 have no unit past 99 in their c = 3 slot and skip it as a whole warp.
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  float* Xc = s.scratch;
  for (int k0 = 0; k0 < kIn; k0 += kKc3) {
    for (int idx = threadIdx.x; idx < mb * kKc3; idx += kThreads) {
      const int i = idx / kKc3, kk = idx % kKc3;
      Xc[idx] = xs[int64_t(s.row[i]) * kIn + k0 + kk];
    }
    __syncthreads();
    float acc[4][7];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int e = 0; e < 7; ++e) acc[c][e] = 0.f;
    const bool c3 = ty + 96 < kHid;
    for (int i = 0; i < mb; ++i) {
      float xv[7], dv[4];
#pragma unroll
      for (int e = 0; e < 7; ++e) xv[e] = Xc[i * kKc3 + tx + 8 * e];
#pragma unroll
      for (int c = 0; c < 3; ++c) dv[c] = s.A[i * kLdA + ty + 32 * c];
      dv[3] = c3 ? s.A[i * kLdA + ty + 96] : 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int e = 0; e < 7; ++e) acc[c][e] = fmaf(dv[c], xv[e], acc[c][e]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = ty + 32 * c;
      if (j >= kHid) continue;
#pragma unroll
      for (int e = 0; e < 7; ++e) g[j * kIn + k0 + tx + 8 * e] = acc[c][e];
    }
    __syncthreads();
  }
}

// Evaluation: CTA (t, b) runs test batch t of problem b's test set (rows [t m, min(t m + m, n_test))) and writes the
// batch's mean NLL (a fp32 sum over rows in order, divided by the row count) and its correct count to the workspace.
template <int RT>
__global__ void __launch_bounds__(kThreads, 2)
evaluate_kernel(const float* __restrict__ weights, const float* __restrict__ x, const int64_t* __restrict__ y,
                int n_sets, int n_test, const int* __restrict__ data_index, int m, float* __restrict__ batch_loss,
                int* __restrict__ batch_correct) {
  const int t = blockIdx.x, b = blockIdx.y, nb = gridDim.x;
  const int set = data_index[b];
  if (set < 0 || set >= n_sets) return;
  extern __shared__ float smem[];
  const Smem s = carve(smem);
  const float* w = weights + int64_t(b) * kD;
  const float* xs = x + int64_t(set) * n_test * kIn;
  const int64_t* ys = y + int64_t(set) * n_test;
  const int lo = t * m, mb = min(lo + m, n_test) - lo;
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    s.row[i] = lo + i;
    s.label[i] = static_cast<int>(ys[lo + i]);
  }
  stage_w2(w, s);
  __syncthreads();
  forward_hidden<RT>(xs, w, mb, s);
  __syncthreads();
  forward_logits(w, mb, s);
  __syncthreads();
  // per row: P[i][0] <- NLL, P[i][1] <- 1 when the argmax (first maximum) is the label
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    float z[kOut], lp[kOut];
#pragma unroll
    for (int c = 0; c < kOut; ++c) z[c] = s.P[i * kOut + c];
    log_softmax_row(z, lp);
    int best = 0;
#pragma unroll
    for (int c = 1; c < kOut; ++c) best = lp[c] > lp[best] ? c : best;
    const int yi = s.label[i];
    s.P[i * kOut] = yi >= 0 && yi < kOut ? -lp[yi] : __int_as_float(0x7fc00000);   // a label outside 0..9: NaN
    s.P[i * kOut + 1] = best == yi ? 1.f : 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float loss = 0.f;
    int correct = 0;
    for (int i = 0; i < mb; ++i) {
      loss += s.P[i * kOut];
      correct += s.P[i * kOut + 1] != 0.f;
    }
    batch_loss[int64_t(b) * nb + t] = loss / static_cast<float>(mb);
    batch_correct[int64_t(b) * nb + t] = correct;
  }
}

// loss_sum[slot][b] = sum_t batch_loss[b][t] in float64, t in order (harness.main's `test_loss += ....item()`);
// correct[slot][b] = sum_t batch_correct[b][t].  A slot outside [0, n_slots) writes nothing.
__global__ void evaluate_finish_kernel(int batch, int nb, const int* __restrict__ data_index, int n_sets,
                                       const float* __restrict__ batch_loss, const int* __restrict__ batch_correct,
                                       const int* __restrict__ slot, int n_slots, double* __restrict__ loss_sum,
                                       int* __restrict__ correct) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int sl = *slot;
  if (b >= batch || sl < 0 || sl >= n_slots) return;
  const int set = data_index[b];
  if (set < 0 || set >= n_sets) return;
  double loss = 0.0;
  int c = 0;
  for (int t = 0; t < nb; ++t) {
    loss += static_cast<double>(batch_loss[int64_t(b) * nb + t]);
    c += batch_correct[int64_t(b) * nb + t];
  }
  loss_sum[int64_t(sl) * batch + b] = loss;
  correct[int64_t(sl) * batch + b] = c;
}

static int smem_done_grad[8][kMaxDevices];
static int smem_done_eval[8][kMaxDevices];

template <int RT>
static int launch_grad(dim3 grid, cudaStream_t stream, const float* weights, const float* x, const int64_t* y,
                       int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                       int n_max, int m, const int* epoch, float* G, int64_t batch_stride, int64_t ld) {
  AFL_CUDA(ensure_dyn_smem(client_grad_kernel<RT>, static_cast<int>(kSmemBytes), smem_done_grad[RT - 1]));
  client_grad_kernel<RT><<<grid, kThreads, kSmemBytes, stream>>>(weights, x, y, n_sets, n_rows, set_len, data_index,
                                                                  rows, n_max, m, epoch, G, batch_stride, ld);
  AFL_LAUNCH_CHECK("client_grad_kernel");
  return AFL_OK;
}

template <int RT>
static int launch_eval(dim3 grid, cudaStream_t stream, const float* weights, const float* x, const int64_t* y,
                       int n_sets, int n_test, const int* data_index, int m, float* batch_loss, int* batch_correct) {
  AFL_CUDA(ensure_dyn_smem(evaluate_kernel<RT>, static_cast<int>(kSmemBytes), smem_done_eval[RT - 1]));
  evaluate_kernel<RT><<<grid, kThreads, kSmemBytes, stream>>>(weights, x, y, n_sets, n_test, data_index, m,
                                                               batch_loss, batch_correct);
  AFL_LAUNCH_CHECK("evaluate_kernel");
  return AFL_OK;
}

#define AFL_MNIST_BY_ROWS(RT_EXPR, FN, ...)                                                   \
  switch (RT_EXPR) {                                                                          \
    case 1: return FN<1>(__VA_ARGS__);                                                        \
    case 2: return FN<2>(__VA_ARGS__);                                                        \
    case 3: return FN<3>(__VA_ARGS__);                                                        \
    case 4: return FN<4>(__VA_ARGS__);                                                        \
    case 5: return FN<5>(__VA_ARGS__);                                                        \
    case 6: return FN<6>(__VA_ARGS__);                                                        \
    case 7: return FN<7>(__VA_ARGS__);                                                        \
    default: return FN<8>(__VA_ARGS__);                                                       \
  }

static int run_eval(dim3 grid, cudaStream_t stream, const float* weights, const float* x, const int64_t* y, int n_sets,
                    int n_test, const int* data_index, int m, float* batch_loss, int* batch_correct) {
  AFL_MNIST_BY_ROWS((m + 15) / 16, launch_eval, grid, stream, weights, x, y, n_sets, n_test, data_index, m, batch_loss,
                    batch_correct)
}

static int check_common(const char* who, int batch, int64_t d, int n_sets, int n_rows, int m) {
  if (batch < 1 || n_sets < 1 || n_rows < 1 || m < 1) {
    set_error("%s: batch, n_sets, the set size and m must be >= 1 (got %d, %d, %d, %d)", who, batch, n_sets, n_rows, m);
    return AFL_ERR_BAD_ARG;
  }
  if (d != kD) {
    set_error("%s: the MnistNet layout has D = %lld parameters (got %lld)", who, static_cast<long long>(kD),
              static_cast<long long>(d));
    return AFL_ERR_UNSUPPORTED;
  }
  if (m > kMaxBatch) { set_error("%s: batch size m <= %d (got %d)", who, kMaxBatch, m); return AFL_ERR_UNSUPPORTED; }
  if (batch > 65535) { set_error("%s: batch <= 65535 problems (got %d)", who, batch); return AFL_ERR_UNSUPPORTED; }
  return AFL_OK;
}

static int client_grads(const char* who, const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                        int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows, int n, int m,
                        const int* epoch, float* G, int64_t batch_stride, int64_t ld, void* stream) {
  if (!weights || !x || !y || !data_index || !rows || !epoch || !G) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = check_common(who, batch, d, n_sets, n_rows, m)) return rc;
  if (n < 1 || n > 1024) { set_error("%s: 1 <= n <= 1024 clients per problem (got %d)", who, n); return n < 1 ? AFL_ERR_BAD_ARG : AFL_ERR_UNSUPPORTED; }
  if (n > n_rows) { set_error("%s: n (%d) exceeds the training set size (%d)", who, n, n_rows); return AFL_ERR_BAD_ARG; }
  if (ld < d || (batch > 1 && batch_stride < (n - 1) * ld + d)) {
    set_error("%s: ld (%lld) < d or batch_stride (%lld) makes problems overlap", who, static_cast<long long>(ld),
              static_cast<long long>(batch_stride));
    return AFL_ERR_BAD_ARG;
  }
  const dim3 grid(n, batch);
  AFL_MNIST_BY_ROWS((m + 15) / 16, launch_grad, grid, static_cast<cudaStream_t>(stream), weights, x, y, n_sets, n_rows,
                    set_len, data_index, rows, n, m, epoch, G, batch_stride, ld)
}

static int64_t eval_batches(int n_test, int m) { return (int64_t(n_test) + m - 1) / m; }

}  // namespace mnist
}  // namespace afl

using namespace afl;

extern "C" {

int afl_mnist_client_grads(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                           int n_train, const int* data_index, const int* rows, int n, int m, const int* epoch,
                           float* G, int64_t batch_stride, int64_t ld, void* stream) {
  return mnist::client_grads("afl_mnist_client_grads", weights, batch, d, x, y, n_sets, n_train, nullptr, data_index,
                             rows, n, m, epoch, G, batch_stride, ld, stream);
}

int afl_mnist_client_grads_sets(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                int n, int m, const int* epoch, float* G, int64_t batch_stride, int64_t ld,
                                void* stream) {
  if (!set_len) { set_error("afl_mnist_client_grads_sets: a pointer argument is NULL"); return AFL_ERR_BAD_ARG; }
  return mnist::client_grads("afl_mnist_client_grads_sets", weights, batch, d, x, y, n_sets, n_rows, set_len,
                             data_index, rows, n, m, epoch, G, batch_stride, ld, stream);
}

size_t afl_mnist_evaluate_workspace_bytes(int batch, int n_test, int m) {
  if (batch < 1 || n_test < 1 || m < 1) return 0;
  const size_t per = static_cast<size_t>(batch) * mnist::eval_batches(n_test, m);
  return align_up(per * sizeof(float), 256) + align_up(per * sizeof(int), 256);
}

int afl_mnist_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                       int n_test, const int* data_index, int m, const int* slot_index, int n_slots, double* loss_sum,
                       int* correct, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "afl_mnist_evaluate";
  if (!weights || !x || !y || !data_index || !slot_index || !loss_sum || !correct || !workspace) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = mnist::check_common(who, batch, d, n_sets, n_test, m)) return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  const size_t need = afl_mnist_evaluate_workspace_bytes(batch, n_test, m);
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 256) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, workspace_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  const int64_t nb = mnist::eval_batches(n_test, m);
  if (nb > 65535) { set_error("%s: at most 65535 test batches (got %lld)", who, static_cast<long long>(nb)); return AFL_ERR_UNSUPPORTED; }
  float* batch_loss = static_cast<float*>(workspace);
  int* batch_correct = reinterpret_cast<int*>(static_cast<char*>(workspace) +
                                              align_up(static_cast<size_t>(batch) * nb * sizeof(float), 256));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(static_cast<unsigned>(nb), batch);
  if (int rc = mnist::run_eval(grid, st, weights, x, y, n_sets, n_test, data_index, m, batch_loss, batch_correct))
    return rc;
  mnist::evaluate_finish_kernel<<<(batch + 127) / 128, 128, 0, st>>>(batch, static_cast<int>(nb), data_index, n_sets,
                                                                     batch_loss, batch_correct, slot_index, n_slots, loss_sum,
                                                                     correct);
  AFL_LAUNCH_CHECK("evaluate_finish_kernel");
  return AFL_OK;
}

}  // extern "C"
