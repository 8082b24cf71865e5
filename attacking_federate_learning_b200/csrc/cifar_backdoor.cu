// The backdoor attacker's Cifar10Net training and backdoor test for a batch of problems: the model half of a CIFAR10
// backdoor sweep epoch (sweep.py with dataset='CIFAR10').
//
// backdoor_train_kernel is harness.BackdoorTrainer.train (backdoor.py:108-159) on harness.Cifar10Net for every
// attacking problem, with backdoor_train.cu's activity condition, status codes and update arithmetic (DESIGN 2.8): the
// BEFORE test on the problem's backdoor set, then mal_epochs passes of minibatch SGD over the set, each step from a
// fresh optimiser: p <- p - 0.1 (g + 1e-4 p), g the gradient of NLL(mean) + alpha * sum over the ten tensors of
// MSE(p, p0).  backdoor_test_kernel and backdoor_test_finish_kernel are BackdoorTrainer.test('POST') (main.py:91-95)
// at any weights.
//
// One 256-thread CTA runs one problem for the whole training call, with cifar_net.cuh's chunked forward and backward
// pass (DESIGN 2.9): each step's NLL gradient is accumulated, 16 rows at a time, into the problem's row of a gradient
// workspace exactly as client_grad_kernel accumulates a client's gradient into its row of G, so a step's gradient is
// bit for bit afl_cifar10_client_grads' on the same rows.  After a barrier the update reads that row and rewrites the
// parameters being trained, which are the output vector itself.  Every sum is one thread's loop in a fixed order and
// nothing is atomic, so a problem's result depends only on its own initial vector, its set and the hyperparameters.
// Full fp32 FFMA throughout (no TF32).
#include "cifar_net.cuh"

namespace afl {
namespace cifar {

constexpr int kMaxRows = 200;                       // BackdoorTrainer's minibatch and test batch
constexpr size_t kSmemRows = smem_bytes(kMaxRows);

// mse_loss's backward factor 2 / numel of the tensor holding parameter o (ParamLayout order).
__device__ __forceinline__ float mse_norm(int o) {
  return o < kOffB1c ? 2.f / 432   : o < kOffW2c ? 2.f / 16  : o < kOffB2c ? 2.f / 16'384 : o < kOffW1 ? 2.f / 64
       : o < kOffB1  ? 2.f / 24'576 : o < kOffW2  ? 2.f / 384 : o < kOffB2  ? 2.f / 73'728 : o < kOffW3 ? 2.f / 192
       : o < kOffB3  ? 2.f / 1'920  : 2.f / 10;
}

// Rows lo .. lo + mb of the set into s.row / s.label.  Ends at a barrier.
__device__ __forceinline__ void stage_rows(const int64_t* __restrict__ ys, int lo, int mb, const Smem& s) {
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    s.row[i] = lo + i;
    s.label[i] = static_cast<int>(ys[lo + i]);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1)
backdoor_train_kernel(const float* __restrict__ initial, float* out, const float* __restrict__ x,
                      const int64_t* __restrict__ y, int n_sets, int max_len, const int* __restrict__ set_len,
                      const int* __restrict__ data_index, const int* __restrict__ fs, const double* __restrict__ zs,
                      int* status, float alpha, int epochs, int m, float* __restrict__ grad) {
  const int b = blockIdx.x, t = threadIdx.x;
  if (fs[b] <= 0 || zs[b] == 0.0 || status[b] != AFL_OK) return;       // batched.backdoor_rows' attacking problems
  const int set = data_index[b];
  const int len = set >= 0 && set < n_sets ? set_len[set] : 0;
  __syncthreads();                                                      // every thread has read status[b]
  if (len < 1 || len > max_len) {
    if (t == 0) status[b] = AFL_ERR_BAD_ARG;
    return;
  }
  extern __shared__ float smem[];
  const Smem s = carve(smem, kMaxRows);
  const float* xs = x + int64_t(set) * max_len * kImg;
  const int64_t* ys = y + int64_t(set) * max_len;
  const float* p0 = initial + int64_t(b) * kD;
  float* p = out + int64_t(b) * kD;
  float* g = grad + int64_t(b) * kD;
  // the output starts as initial; p0 - p0 is NaN where initial holds a NaN or an infinity (the first dist loss)
  bool bad = false;
  for (int c = t; c < kD; c += kThreads) {
    const float v = p0[c];
    p[c] = v;
    if (__fsub_rn(v, v) != 0.f) bad = true;
  }
  // BEFORE: the test at initial (read-only here, so through the read-only cache); 100 % already returns initial
  stage_conv1<true>(p0, s);
  int correct = 0;
  for (int lo = 0; lo < len; lo += m) {
    const int mb = min(m, len - lo);
    stage_rows(ys, lo, mb, s);
    for (int c0 = 0; c0 < mb; c0 += kS) {
      const int mc = min(kS, mb - c0);
      forward_chunk<true>(xs, p0, c0, mc, s);
      bool hit = false;
      if (t < mc) train::row_head(s.Z + t * kOut, s.label[c0 + t], &hit);
      correct += __syncthreads_count(hit);
    }
  }
  if (correct >= len) return;
  const bool dist = alpha > 0.f;
  bool dist_nan = __syncthreads_or(bad);
  for (int e = 0; e < epochs; ++e) {
    for (int lo = 0; lo < len; lo += m) {
      const int mb = min(m, len - lo);
      if (dist && dist_nan) {                                           // "Got nan dist loss"
        if (t == 0) status[b] = AFL_ERR_NAN_DIST_LOSS;
        return;
      }
      stage_conv1<false>(p, s);
      stage_rows(ys, lo, mb, s);
      // the step's NLL gradient into g, chunk by chunk (client_grad_kernel's loop); each row's loss is read from the
      // chunk's logits by the thread that turns them into delta3, before backward_chunk does
      bool nan_row = false;
      for (int c0 = 0; c0 < mb; c0 += kS) {
        const int mc = min(kS, mb - c0);
        forward_chunk<false>(xs, p, c0, mc, s);
        if (t < mc) {
          bool hit;
          const float l = train::row_head(s.Z + t * kOut, s.label[c0 + t], &hit);
          nan_row |= l != l;
        }
        backward_chunk<false>(xs, p, c0, mc, mb, c0 == 0, s, g);
      }
      if (__syncthreads_or(nan_row)) {                                  // "Got nan loss": p keeps the last step's
        if (t == 0) status[b] = AFL_ERR_NAN_LOSS;
        return;
      }
      bad = false;
      for (int o = t; o < kD; o += kThreads) p[o] = train::sgd(p[o], p0[o], g[o], mse_norm(o), alpha, dist, &bad);
      dist_nan = __syncthreads_or(bad);                                 // also: every update lands before the next read
    }
  }
}

// BackdoorTrainer.test's batch t = blockIdx.x of problem b = blockIdx.y at weights[b] (rows [t m, min(t m + m, len))
// of its set): the batch's mean NLL (a fp32 sum over rows in order, divided by the row count) and its correct count
// into the workspace.  A batch past the set, or an out-of-range set index, length or slot, writes nothing.
__global__ void __launch_bounds__(kThreads, 2)
backdoor_test_kernel(const float* __restrict__ weights, const float* __restrict__ x, const int64_t* __restrict__ y,
                     int n_sets, int max_len, const int* __restrict__ set_len, const int* __restrict__ data_index,
                     int m, const int* __restrict__ slot, int n_slots, float* __restrict__ batch_loss,
                     int* __restrict__ batch_correct) {
  const int t = blockIdx.x, b = blockIdx.y, nb = gridDim.x;
  const int set = data_index[b], sl = *slot;
  const int len = set >= 0 && set < n_sets ? set_len[set] : 0;
  const int lo = t * m;
  if (len < 1 || len > max_len || lo >= len || sl < 0 || sl >= n_slots) return;
  extern __shared__ float smem[];
  const Smem s = carve(smem, kMaxRows);
  const float* w = weights + int64_t(b) * kD;
  const float* xs = x + int64_t(set) * max_len * kImg;
  const int mb = min(m, len - lo);
  stage_conv1<true>(w, s);
  stage_rows(y + int64_t(set) * max_len, lo, mb, s);
  for (int c0 = 0; c0 < mb; c0 += kS) {
    const int mc = min(kS, mb - c0);
    forward_chunk<true>(xs, w, c0, mc, s);
    if (threadIdx.x < mc) {
      bool hit;
      s.nll[c0 + threadIdx.x] = train::row_head(s.Z + threadIdx.x * kOut, s.label[c0 + threadIdx.x], &hit);
      s.hit[c0 + threadIdx.x] = hit ? 1.f : 0.f;
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

// loss_sum[slot][b] = the float64 sum of problem b's batch means, batches in order (BackdoorTrainer.test's
// `loss += ....item()`); correct[slot][b] = the sum of its batch counts.  Same write rule as backdoor_test_kernel.
__global__ void backdoor_test_finish_kernel(int batch, int nb, int n_sets, int max_len, const int* __restrict__ set_len,
                                            const int* __restrict__ data_index, int m,
                                            const float* __restrict__ batch_loss, const int* __restrict__ batch_correct,
                                            const int* __restrict__ slot, int n_slots, double* __restrict__ loss_sum,
                                            int* __restrict__ correct) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const int set = data_index[b], sl = *slot;
  const int len = set >= 0 && set < n_sets ? set_len[set] : 0;
  if (len < 1 || len > max_len || sl < 0 || sl >= n_slots) return;
  double loss = 0.0;
  int c = 0;
  for (int t = 0; t < (len + m - 1) / m; ++t) {
    loss += static_cast<double>(batch_loss[int64_t(b) * nb + t]);
    c += batch_correct[int64_t(b) * nb + t];
  }
  loss_sum[int64_t(sl) * batch + b] = loss;
  correct[int64_t(sl) * batch + b] = c;
}

static int smem_done_bd_train[kMaxDevices];
static int smem_done_bd_test[kMaxDevices];

}  // namespace cifar
}  // namespace afl

using namespace afl;

extern "C" {

size_t afl_cifar10_backdoor_train_workspace_bytes(int batch) {
  if (batch < 1) return 0;
  return static_cast<size_t>(batch) * cifar::kD * sizeof(float);
}

int afl_cifar10_backdoor_train(const float* initial, float* out, int batch, int64_t d, const float* x,
                               const int64_t* y, int n_sets, int max_len, const int* set_len, const int* data_index,
                               const int* f, const double* z, int* status, double alpha, int mal_epochs, int m,
                               void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "afl_cifar10_backdoor_train";
  if (!initial || !out || !x || !y || !set_len || !data_index || !f || !z || !status || !workspace) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = train::check_common(who, "Cifar10Net", cifar::kD, cifar::kMaxRows, "max_len", batch, d, n_sets,
                                   max_len, m))
    return rc;
  if (mal_epochs < 0 || alpha != alpha) {
    set_error("%s: mal_epochs must be >= 0 and alpha a number (got %d, %g)", who, mal_epochs, alpha);
    return AFL_ERR_BAD_ARG;
  }
  const size_t need = afl_cifar10_backdoor_train_workspace_bytes(batch);
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % sizeof(float)) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, workspace_bytes, need);
    return AFL_ERR_BAD_ARG;
  }
  const size_t span = static_cast<size_t>(batch) * cifar::kD * sizeof(float);
  if (train::overlap(initial, span, out, span) || train::overlap(workspace, need, out, span) ||
      train::overlap(workspace, need, initial, span)) {
    set_error("%s: out, initial and the workspace must not overlap", who);
    return AFL_ERR_BAD_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(cifar::backdoor_train_kernel, static_cast<int>(cifar::kSmemRows),
                           cifar::smem_done_bd_train));
  ProfScope ps("cifar10_backdoor_train", st);
  cifar::backdoor_train_kernel<<<batch, cifar::kThreads, cifar::kSmemRows, st>>>(
      initial, out, x, y, n_sets, max_len, set_len, data_index, f, z, status, static_cast<float>(alpha), mal_epochs, m,
      static_cast<float*>(workspace));
  AFL_LAUNCH_CHECK("cifar10_backdoor_train_kernel");
  return AFL_OK;
}

size_t afl_cifar10_backdoor_test_workspace_bytes(int batch, int max_len, int m) {
  return train::eval_workspace_bytes(batch, max_len, m);
}

int afl_cifar10_backdoor_test(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                              int max_len, const int* set_len, const int* data_index, int m, const int* slot_index,
                              int n_slots, double* loss_sum, int* correct, void* workspace, size_t workspace_bytes,
                              void* stream) {
  const char* who = "afl_cifar10_backdoor_test";
  if (!weights || !x || !y || !set_len || !data_index || !slot_index || !loss_sum || !correct || !workspace) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = train::check_common(who, "Cifar10Net", cifar::kD, cifar::kMaxRows, "max_len", batch, d, n_sets,
                                   max_len, m))
    return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  train::EvalWorkspace ws;
  if (int rc = train::carve_eval_workspace(who, workspace, workspace_bytes, batch, max_len, m, AFL_ERR_BAD_ARG, &ws))
    return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(cifar::backdoor_test_kernel, static_cast<int>(cifar::kSmemRows), cifar::smem_done_bd_test));
  cifar::backdoor_test_kernel<<<dim3(ws.nb, batch), cifar::kThreads, cifar::kSmemRows, st>>>(
      weights, x, y, n_sets, max_len, set_len, data_index, m, slot_index, n_slots, ws.batch_loss, ws.batch_correct);
  AFL_LAUNCH_CHECK("cifar10_backdoor_test_kernel");
  cifar::backdoor_test_finish_kernel<<<(batch + 127) / 128, 128, 0, st>>>(
      batch, ws.nb, n_sets, max_len, set_len, data_index, m, ws.batch_loss, ws.batch_correct, slot_index, n_slots,
      loss_sum, correct);
  AFL_LAUNCH_CHECK("cifar10_backdoor_test_finish_kernel");
  return AFL_OK;
}

}  // extern "C"
