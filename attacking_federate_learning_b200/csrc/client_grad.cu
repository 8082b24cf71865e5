// Batched MnistNet client gradients and test-set evaluation: the training half of a sweep epoch (sweep.py).
//
// One CTA runs one client (grid x = client, y = problem): it finds its minibatch's rows from the device epoch
// counter, runs the forward pass, the NLL(mean) backward and writes the gradient straight into its row of the client
// matrix.  Every sum is a sequential loop of one thread in a fixed order and nothing is atomic, so a client's gradient
// depends only on its weights, its rows and m.  Full fp32 FFMA throughout (the reference trains in fp32; no TF32).
// The net's layout and passes live in mnist_net.cuh, which the backdoor attacker's trainer (backdoor_train.cu) shares.
#include "mnist_net.cuh"

namespace afl {
namespace mnist {

// 256 threads, up to 128 rows (16 row lanes x RT <= 8 rows), 16-column forward k-chunks (784 = 49 x 16) and 56-column
// weight-gradient chunks (784 = 14 x 56: 8 column lanes x 7 columns).  90.5 KB of shared memory, two CTAs per SM.
using Geo = Geometry<256, 128, 16>;
constexpr int kThreads = Geo::kThreads, kMaxBatch = Geo::kRows;
constexpr size_t kSmemBytes = Geo::kSmemBytes;

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
  const Smem s = carve<Geo>(smem);
  const float* w = weights + int64_t(b) * kD;
  const float* xs = x + int64_t(set) * n_rows * kIn;
  const int64_t* ys = y + int64_t(set) * n_rows;
  int mb;
  const int lo = train::batch_start(n_train, n, u, m, *epoch, &mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) s.label[i] = static_cast<int>(ys[u + n * (lo + i)]);
  const float* x0 = xs + (u + int64_t(n) * lo) * kIn;             // row i of the minibatch is shard row u + n (lo + i)
  const int64_t pitch = int64_t(n) * kIn;
  stage_w2<Geo>(w, s);
  __syncthreads();
  forward_hidden<Geo, RT>(x0, pitch, w, mb, s);
  __syncthreads();
  forward_logits<Geo>(w, mb, s);
  __syncthreads();
  const float fmb = static_cast<float>(mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    float lp[kOut];
    train::log_softmax_row(s.P + i * kOut, lp);
    train::row_delta(lp, s.label[i], fmb, s.P + i * kOut);
  }
  __syncthreads();
  float* g = G + int64_t(b) * batch_stride + int64_t(u) * ld;
  for (int idx = threadIdx.x; idx < kOut * kHid + kOut; idx += kThreads) {
    if (idx < kOut * kHid) g[kOffW2 + idx] = fc2_weight_grad(idx, mb, s);
    else g[kOffB2 + idx - kOut * kHid] = fc2_bias_grad(idx - kOut * kHid, mb, s);
  }
  __syncthreads();
  backward_hidden<Geo>(mb, s);
  __syncthreads();
  for (int j = threadIdx.x; j < kHid; j += kThreads) {
    float acc = 0.f;
    for (int i = 0; i < mb; ++i) acc += s.A[i * kLdA + j];
    g[kOffB1 + j] = acc;
  }
  const int tx = threadIdx.x % Geo::kColLanes, ty = threadIdx.x / Geo::kColLanes;
  for (int k0 = 0; k0 < kIn; k0 += Geo::kKc3) {
    float acc[4][7];
    fc1_weight_grad<Geo>(x0, pitch, k0, mb, s, acc);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = ty + 32 * c;
      if (j >= kHid) continue;
#pragma unroll
      for (int e = 0; e < 7; ++e) g[j * kIn + k0 + tx + Geo::kColLanes * e] = acc[c][e];
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
  const Smem s = carve<Geo>(smem);
  const float* w = weights + int64_t(b) * kD;
  const float* xs = x + int64_t(set) * n_test * kIn;
  const int64_t* ys = y + int64_t(set) * n_test;
  const int lo = t * m, mb = min(lo + m, n_test) - lo;
  for (int i = threadIdx.x; i < mb; i += kThreads) s.label[i] = static_cast<int>(ys[lo + i]);
  stage_w2<Geo>(w, s);
  __syncthreads();
  forward_hidden<Geo, RT>(xs + int64_t(lo) * kIn, kIn, w, mb, s);
  __syncthreads();
  forward_logits<Geo>(w, mb, s);
  __syncthreads();
  // per row: P[i][0] <- NLL, P[i][1] <- 1 when the argmax is the label
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    bool hit;
    s.P[i * kOut] = train::row_head(s.P + i * kOut, s.label[i], &hit);
    s.P[i * kOut + 1] = hit ? 1.f : 0.f;
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

static int client_grads(const char* who, const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                        int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows, int n, int m,
                        const int* epoch, float* G, int64_t batch_stride, int64_t ld, void* stream) {
  if (int rc = train::check_client_grads(who, "MnistNet", kD, kMaxBatch, weights, batch, d, x, y, n_sets, n_rows,
                                         data_index, rows, n, m, epoch, G, batch_stride, ld))
    return rc;
  const dim3 grid(n, batch);
  AFL_MNIST_BY_ROWS((m + 15) / 16, launch_grad, grid, static_cast<cudaStream_t>(stream), weights, x, y, n_sets, n_rows,
                    set_len, data_index, rows, n, m, epoch, G, batch_stride, ld)
}

}  // namespace mnist

namespace train {

// loss_sum[slot][b] and correct[slot][b] from the per-batch workspace (evaluate_finish in train_common.cuh).  A slot
// outside [0, n_slots) writes nothing.
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

int evaluate_finish(cudaStream_t stream, int batch, const EvalWorkspace& ws, const int* data_index, int n_sets,
                    const int* slot_index, int n_slots, double* loss_sum, int* correct) {
  evaluate_finish_kernel<<<(batch + 127) / 128, 128, 0, stream>>>(batch, ws.nb, data_index, n_sets, ws.batch_loss,
                                                                  ws.batch_correct, slot_index, n_slots, loss_sum,
                                                                  correct);
  AFL_LAUNCH_CHECK("evaluate_finish_kernel");
  return AFL_OK;
}

}  // namespace train
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
  return train::eval_workspace_bytes(batch, n_test, m);
}

int afl_mnist_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                       int n_test, const int* data_index, int m, const int* slot_index, int n_slots, double* loss_sum,
                       int* correct, void* workspace, size_t workspace_bytes, void* stream) {
  train::EvalWorkspace ws;
  if (int rc = train::check_evaluate("afl_mnist_evaluate", "MnistNet", mnist::kD, mnist::kMaxBatch, weights, batch, d,
                                     x, y, n_sets, n_test, data_index, m, slot_index, n_slots, loss_sum, correct,
                                     workspace, workspace_bytes, &ws))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = mnist::run_eval(dim3(ws.nb, batch), st, weights, x, y, n_sets, n_test, data_index, m, ws.batch_loss,
                               ws.batch_correct))
    return rc;
  return train::evaluate_finish(st, batch, ws, data_index, n_sets, slot_index, n_slots, loss_sum, correct);
}

}  // extern "C"
