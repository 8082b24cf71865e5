// The backdoor attacker's MnistNet training and backdoor test for a batch of problems: the model half of a backdoor
// sweep epoch (sweep.py).
//
// backdoor_train_kernel is harness.BackdoorTrainer.train (backdoor.py:108-159) for every attacking problem: the BEFORE
// test on the problem's backdoor set, then mal_epochs passes of minibatch SGD over the set, each step from a fresh
// optimiser (so the momentum buffer is d_p): p <- p - 0.1 (g + 1e-4 p), g the gradient of NLL(mean) + alpha *
// sum_tensors MSE(p, p0).  backdoor_test_kernel is BackdoorTrainer.test('POST') (main.py:91-95) at any weights.
//
// One 512-thread CTA runs one problem for the whole call: the hidden activations and deltas of a minibatch (up to 200
// rows), fc2 and the staged inputs live in shared memory, and the parameters being trained are the output vector
// itself (fc1's 78,400 weights do not fit in shared memory), updated in place after each step's forward pass has read
// them.  Every sum is one thread's loop in a fixed order and nothing is atomic, so a problem's result depends only on
// its own initial vector, its set and the hyperparameters.  Full fp32 FFMA throughout (no TF32).  The net's layout
// and passes live in mnist_net.cuh, which the client-gradient kernels (client_grad.cu) share.
#include "mnist_net.cuh"

namespace afl {
namespace mnist {

// 512 threads, up to 200 rows (BackdoorTrainer's batch size: 32 row lanes x 7 rows), 28-column forward k-chunks
// (784 = 28 x 28) and 112-column weight-gradient chunks (784 = 7 x 112: 16 column lanes x 7 columns).
using BdGeo = Geometry<512, 200, 28>;
constexpr int kBdThreads = BdGeo::kThreads, kBdRows = BdGeo::kRows, kRT = 7;

// The forward pass of set rows lo .. lo + mb at the parameters w, to the logits in s.P; also stages fc2 and the
// labels.  w may be the vector being trained: it is read through ordinary loads only.  Starts after
// the previous readers of shared memory have passed a barrier; ends at a barrier.
__device__ void forward(const float* __restrict__ xs, const int64_t* __restrict__ ys, int lo, const float* w, int mb,
                        const Smem& s) {
  stage_w2<BdGeo>(w, s);
  for (int i = threadIdx.x; i < mb; i += kBdThreads) s.label[i] = static_cast<int>(ys[lo + i]);
  __syncthreads();
  forward_hidden<BdGeo, kRT>(xs + int64_t(lo) * kIn, kIn, w, mb, s);
  __syncthreads();
  forward_logits<BdGeo>(w, mb, s);
  __syncthreads();
}

// BackdoorTrainer.test on the set's len rows at the parameters w: batches of m rows (the last one shorter).  Returns the
// correct count (every thread); thread 0 also gets the float64 sum of the batches' fp32 mean NLL (rows in order) in
// *loss.  Starts and ends at a barrier.
__device__ int test_set(const float* __restrict__ xs, const int64_t* __restrict__ ys, int len, int m, const float* w,
                        const Smem& s, double* loss) {
  int correct = 0;
  double total = 0.0;
  for (int lo = 0; lo < len; lo += m) {
    const int mb = min(m, len - lo);
    forward(xs, ys, lo, w, mb, s);
    bool hit = false;
    const int i = threadIdx.x;
    if (i < mb) s.P[i * kOut] = train::row_head(s.P + i * kOut, s.label[i], &hit);   // row i's NLL over its logits
    correct += __syncthreads_count(hit);
    if (threadIdx.x == 0) {
      float sum = 0.f;
      for (int r = 0; r < mb; ++r) sum += s.P[r * kOut];
      total += static_cast<double>(sum / static_cast<float>(mb));
    }
  }
  *loss = total;
  return correct;
}

__global__ void __launch_bounds__(kBdThreads, 1)
backdoor_train_kernel(const float* __restrict__ initial, float* out, const float* __restrict__ x,
                      const int64_t* __restrict__ y, int n_sets, int max_len, const int* __restrict__ set_len,
                      const int* __restrict__ data_index, const int* __restrict__ fs, const double* __restrict__ zs,
                      int* status, float alpha, int epochs, int m) {
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
  const Smem s = carve<BdGeo>(smem);
  const float* xs = x + int64_t(set) * max_len * kIn;
  const int64_t* ys = y + int64_t(set) * max_len;
  const float* p0 = initial + int64_t(b) * kD;
  float* p = out + int64_t(b) * kD;
  // the output starts as initial; p0 - p0 is NaN where initial holds a NaN or an infinity (the first dist loss)
  bool bad = false;
  for (int c = t; c < kD; c += kBdThreads) {
    const float v = p0[c];
    p[c] = v;
    if (__fsub_rn(v, v) != 0.f) bad = true;
  }
  double unused;
  if (test_set(xs, ys, len, m, p0, s, &unused) >= len) return;         // BEFORE: 100 % already, initial returned
  const bool dist = alpha > 0.f;
  bool dist_nan = __syncthreads_or(bad);
  for (int e = 0; e < epochs; ++e) {
    for (int lo = 0; lo < len; lo += m) {
      const int mb = min(m, len - lo);
      if (dist && dist_nan) {                                           // "Got nan dist loss"
        if (t == 0) status[b] = AFL_ERR_NAN_DIST_LOSS;
        return;
      }
      forward(xs, ys, lo, p, mb, s);
      bool nan_row = false;
      if (t < mb) {                                                     // row t's loss, then delta2 in place
        float* z = s.P + t * kOut;
        bool hit;
        const float l = train::row_head(z, s.label[t], &hit);
        nan_row = l != l;
        float lp[kOut];
        train::log_softmax_row(z, lp);
        train::row_delta(lp, s.label[t], static_cast<float>(mb), z);
      }
      if (__syncthreads_or(nan_row)) {                                  // "Got nan loss"
        if (t == 0) status[b] = AFL_ERR_NAN_LOSS;
        return;
      }
      // fc2's gradient, kept until delta1 has read the old fc2
      float g2[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int idx = t + q * kBdThreads;
        g2[q] = idx < kOut * kHid          ? fc2_weight_grad(idx, mb, s)
              : idx < kOut * kHid + kOut ? fc2_bias_grad(idx - kOut * kHid, mb, s) : 0.f;
      }
      __syncthreads();
      backward_hidden<BdGeo>(mb, s);
      bad = false;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int idx = t + q * kBdThreads;
        if (idx < kOut * kHid + kOut) {
          const int o = kOffW2 + idx;
          const float norm = idx < kOut * kHid ? 2.f / (kOut * kHid) : 2.f / kOut;
          p[o] = train::sgd(p[o], p0[o], g2[q], norm, alpha, dist, &bad);
        }
      }
      __syncthreads();
      if (t < kHid) {                                                   // fc1.bias: db1[j] = sum_i delta1[i][j]
        float acc = 0.f;
        for (int i = 0; i < mb; ++i) acc += s.A[i * kLdA + t];
        const int o = kOffB1 + t;
        p[o] = train::sgd(p[o], p0[o], acc, 2.f / kHid, alpha, dist, &bad);
      }
      // fc1.weight, updated in place chunk by chunk
      const int tx = t % BdGeo::kColLanes, ty = t / BdGeo::kColLanes;
      for (int k0 = 0; k0 < kIn; k0 += BdGeo::kKc3) {
        float acc[4][7];
        fc1_weight_grad<BdGeo>(xs + int64_t(lo) * kIn, kIn, k0, mb, s, acc);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = ty + 32 * c;
          if (j >= kHid) continue;
#pragma unroll
          for (int e = 0; e < 7; ++e) {
            const int o = j * kIn + k0 + tx + BdGeo::kColLanes * e;
            p[o] = train::sgd(p[o], p0[o], acc[c][e], 2.f / (kHid * kIn), alpha, dist, &bad);
          }
        }
        __syncthreads();
      }
      dist_nan = __syncthreads_or(bad);
    }
  }
}

// BackdoorTrainer.test('POST') of problem b = blockIdx.x at weights[b]: loss_sum[slot][b] (float64 sum of the batches'
// mean NLL) and correct[slot][b].  A problem whose set index or set length is out of range, or a slot outside
// [0, n_slots), writes nothing.
__global__ void __launch_bounds__(kBdThreads, 1)
backdoor_test_kernel(const float* __restrict__ weights, int batch, const float* __restrict__ x,
                     const int64_t* __restrict__ y, int n_sets, int max_len, const int* __restrict__ set_len,
                     const int* __restrict__ data_index, int m, const int* __restrict__ slot, int n_slots,
                     double* __restrict__ loss_sum, int* __restrict__ correct) {
  const int b = blockIdx.x;
  const int set = data_index[b], sl = *slot;
  const int len = set >= 0 && set < n_sets ? set_len[set] : 0;
  if (len < 1 || len > max_len || sl < 0 || sl >= n_slots) return;
  extern __shared__ float smem[];
  const Smem s = carve<BdGeo>(smem);
  double loss;
  const int c = test_set(x + int64_t(set) * max_len * kIn, y + int64_t(set) * max_len, len, m,
                         weights + int64_t(b) * kD, s, &loss);
  if (threadIdx.x == 0) {
    loss_sum[int64_t(sl) * batch + b] = loss;
    correct[int64_t(sl) * batch + b] = c;
  }
}

static int smem_done_train[kMaxDevices];
static int smem_done_test[kMaxDevices];

}  // namespace mnist
}  // namespace afl

using namespace afl;

extern "C" {

int afl_mnist_backdoor_train(const float* initial, float* out, int batch, int64_t d, const float* x, const int64_t* y,
                             int n_sets, int max_len, const int* set_len, const int* data_index, const int* f,
                             const double* z, int* status, double alpha, int mal_epochs, int m, void* stream) {
  const char* who = "afl_mnist_backdoor_train";
  if (!initial || !out || !x || !y || !set_len || !data_index || !f || !z || !status) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = train::check_common(who, "MnistNet", mnist::kD, mnist::kBdRows, "max_len", batch, d, n_sets,
                                   max_len, m))
    return rc;
  if (mal_epochs < 0 || alpha != alpha) {
    set_error("%s: mal_epochs must be >= 0 and alpha a number (got %d, %g)", who, mal_epochs, alpha);
    return AFL_ERR_BAD_ARG;
  }
  const size_t span = static_cast<size_t>(batch) * mnist::kD * sizeof(float);
  if (train::overlap(initial, span, out, span)) { set_error("%s: out overlaps initial", who); return AFL_ERR_BAD_ARG; }
  AFL_CUDA(ensure_dyn_smem(mnist::backdoor_train_kernel, static_cast<int>(mnist::BdGeo::kSmemBytes),
                           mnist::smem_done_train));
  ProfScope ps("backdoor_train", static_cast<cudaStream_t>(stream));
  mnist::backdoor_train_kernel<<<batch, mnist::kBdThreads, mnist::BdGeo::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
      initial, out, x, y, n_sets, max_len, set_len, data_index, f, z, status, static_cast<float>(alpha), mal_epochs, m);
  AFL_LAUNCH_CHECK("backdoor_train_kernel");
  return AFL_OK;
}

int afl_mnist_backdoor_test(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                            int max_len, const int* set_len, const int* data_index, int m, const int* slot_index,
                            int n_slots, double* loss_sum, int* correct, void* stream) {
  const char* who = "afl_mnist_backdoor_test";
  if (!weights || !x || !y || !set_len || !data_index || !slot_index || !loss_sum || !correct) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = train::check_common(who, "MnistNet", mnist::kD, mnist::kBdRows, "max_len", batch, d, n_sets,
                                   max_len, m))
    return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  AFL_CUDA(ensure_dyn_smem(mnist::backdoor_test_kernel, static_cast<int>(mnist::BdGeo::kSmemBytes),
                           mnist::smem_done_test));
  mnist::backdoor_test_kernel<<<batch, mnist::kBdThreads, mnist::BdGeo::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
      weights, batch, x, y, n_sets, max_len, set_len, data_index, m, slot_index, n_slots, loss_sum, correct);
  AFL_LAUNCH_CHECK("backdoor_test_kernel");
  return AFL_OK;
}

}  // extern "C"
