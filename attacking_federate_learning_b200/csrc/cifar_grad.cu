// Batched Cifar10Net client gradients and test-set evaluation: the training half of a CIFAR10 sweep epoch (sweep.py).
//
// The net is harness.Cifar10Net (data_sets.py:33-52) on [3, 32, 32] images:
//   conv1 3->16 k3, relu, maxpool 3 -> conv2 16->64 k4, relu, maxpool 4 -> fc1 64->384, relu -> fc2 384->192, relu
//   -> fc3 192->10 -> log_softmax,
// flattened in ParamLayout order (D = 117,706).  Both pools use floor mode, so pool2 reads only conv2's top-left 4x4
// of 7x7, which reads pool1's 7x7 of 10x10, which reads conv1's 21x21 of 30x30, which reads the input's 23x23 corner:
// the kernels compute that corner alone (DESIGN 2.9).  Every other position has no path to the loss; on finite values
// its contribution to every gradient is an exact zero.
//
// One CTA runs one client (grid x = client, y = problem) in chunks of kS minibatch rows: the chunk's forward pass
// keeps pool1's 7x7 values and window indices, pool2's values and indices, relu(fc1) and relu(fc2) in shared memory,
// its backward pass adds the chunk's rows to the weight gradients in the client's row of the client matrix (the same
// thread owns the same entries in every chunk, so each entry is one sequential sum over the minibatch rows in order).
// Every other sum is also one thread's loop in a fixed order and nothing is atomic, so a client's gradient depends only
// on its weights, its rows and m.  Full fp32 FFMA throughout (no TF32).  MaxPool follows torch's max_pool2d: the index
// of a window is its first maximum in row-major order, a NaN takes the index, and the backward routes the window's
// gradient to that index alone.  The chunk passes and the shared-memory carve live in cifar_net.cuh, which the backdoor
// attacker's trainer (cifar_backdoor.cu) shares.
#include "cifar_net.cuh"

namespace afl {
namespace cifar {

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
  const float* xs = x + int64_t(set) * n_rows * kImg;
  const int64_t* ys = y + int64_t(set) * n_rows;
  int mb;
  const int lo = train::batch_start(n_train, n, u, m, *epoch, &mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    const int r = u + n * (lo + i);
    s.row[i] = r;
    s.label[i] = static_cast<int>(ys[r]);
  }
  stage_conv1<true>(w, s);
  __syncthreads();
  float* g = G + int64_t(b) * batch_stride + int64_t(u) * ld;
  for (int c0 = 0; c0 < mb; c0 += kS) {
    const int mc = min(kS, mb - c0);
    forward_chunk<true>(xs, w, c0, mc, s);
    backward_chunk<true>(xs, w, c0, mc, mb, c0 == 0, s, g);
  }
}

// Evaluation: CTA (t, b) runs test batch t of problem b's test set (rows [t m, min(t m + m, n_test))) and writes the
// batch's mean NLL (a fp32 sum over rows in order, divided by the row count) and its correct count to the workspace.
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
  const float* xs = x + int64_t(set) * n_test * kImg;
  const int64_t* ys = y + int64_t(set) * n_test;
  const int lo = t * m, mb = min(lo + m, n_test) - lo;
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    s.row[i] = lo + i;
    s.label[i] = static_cast<int>(ys[lo + i]);
  }
  stage_conv1<true>(w, s);
  __syncthreads();
  for (int c0 = 0; c0 < mb; c0 += kS) {
    const int mc = min(kS, mb - c0);
    forward_chunk<true>(xs, w, c0, mc, s);
    // per row: its NLL, and 1 when the argmax is the label
    for (int i = threadIdx.x; i < mc; i += kThreads) {
      bool hit;
      s.nll[c0 + i] = train::row_head(s.Z + i * kOut, s.label[c0 + i], &hit);
      s.hit[c0 + i] = hit ? 1.f : 0.f;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float loss = 0.f;
    int correct = 0;
    for (int i = 0; i < mb; ++i) {
      loss += s.nll[i];
      correct += s.hit[i] != 0.f;
    }
    batch_loss[int64_t(b) * nb + t] = loss / static_cast<float>(mb);
    batch_correct[int64_t(b) * nb + t] = correct;
  }
}

static int smem_done_grad[kMaxDevices];
static int smem_done_eval[kMaxDevices];

static int client_grads(const char* who, const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                        int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows, int n, int m,
                        const int* epoch, float* G, int64_t batch_stride, int64_t ld, void* stream) {
  if (int rc = train::check_client_grads(who, "Cifar10Net", kD, kMaxBatch, weights, batch, d, x, y, n_sets, n_rows,
                                         data_index, rows, n, m, epoch, G, batch_stride, ld))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(client_grad_kernel, static_cast<int>(kSmemBytes), smem_done_grad));
  client_grad_kernel<<<dim3(n, batch), kThreads, kSmemBytes, st>>>(
      weights, x, y, n_sets, n_rows, set_len, data_index, rows, n, m, epoch, G, batch_stride, ld);
  AFL_LAUNCH_CHECK("cifar_client_grad_kernel");
  return AFL_OK;
}

}  // namespace cifar
}  // namespace afl

using namespace afl;

extern "C" {

int afl_cifar10_client_grads(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                             int n_train, const int* data_index, const int* rows, int n, int m, const int* epoch,
                             float* G, int64_t batch_stride, int64_t ld, void* stream) {
  return cifar::client_grads("afl_cifar10_client_grads", weights, batch, d, x, y, n_sets, n_train, nullptr, data_index,
                             rows, n, m, epoch, G, batch_stride, ld, stream);
}

int afl_cifar10_client_grads_sets(const float* weights, int batch, int64_t d, const float* x, const int64_t* y,
                                  int n_sets, int n_rows, const int* set_len, const int* data_index, const int* rows,
                                  int n, int m, const int* epoch, float* G, int64_t batch_stride, int64_t ld,
                                  void* stream) {
  if (!set_len) { set_error("afl_cifar10_client_grads_sets: a pointer argument is NULL"); return AFL_ERR_BAD_ARG; }
  return cifar::client_grads("afl_cifar10_client_grads_sets", weights, batch, d, x, y, n_sets, n_rows, set_len,
                             data_index, rows, n, m, epoch, G, batch_stride, ld, stream);
}

size_t afl_cifar10_evaluate_workspace_bytes(int batch, int n_test, int m) {
  return train::eval_workspace_bytes(batch, n_test, m);
}

int afl_cifar10_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                         int n_test, const int* data_index, int m, const int* slot_index, int n_slots, double* loss_sum,
                         int* correct, void* workspace, size_t workspace_bytes, void* stream) {
  train::EvalWorkspace ws;
  if (int rc = train::check_evaluate("afl_cifar10_evaluate", "Cifar10Net", cifar::kD, cifar::kMaxBatch, weights, batch,
                                     d, x, y, n_sets, n_test, data_index, m, slot_index, n_slots, loss_sum, correct,
                                     workspace, workspace_bytes, &ws))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(cifar::evaluate_kernel, static_cast<int>(cifar::kSmemBytes), cifar::smem_done_eval));
  cifar::evaluate_kernel<<<dim3(ws.nb, batch), cifar::kThreads, cifar::kSmemBytes, st>>>(
      weights, x, y, n_sets, n_test, data_index, m, ws.batch_loss, ws.batch_correct);
  AFL_LAUNCH_CHECK("cifar_evaluate_kernel");
  return train::evaluate_finish(st, batch, ws, data_index, n_sets, slot_index, n_slots, loss_sum, correct);
}

}  // extern "C"
