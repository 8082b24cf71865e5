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
// its own initial vector, its set and the hyperparameters.  Full fp32 FFMA throughout (no TF32).
#include "afl_common.cuh"

namespace afl {
namespace backdoor {

constexpr int kIn = 784, kHid = 100, kOut = 10;
constexpr int64_t kD = int64_t(kHid) * kIn + kHid + kOut * kHid + kOut;        // 79,510
constexpr int kOffB1 = kHid * kIn, kOffW2 = kOffB1 + kHid;
constexpr int kThreads = 512;
constexpr int kMaxBatch = 200;          // minibatch rows a CTA holds: BackdoorTrainer's batch size
constexpr int kRT = 7;                  // forward: 32 row lanes x 7 rows (224 >= 200)
constexpr int kHidPad = 112;            // forward: 16 unit lanes x 7 hidden units
constexpr int kKc1 = 28;                // forward k-chunk (784 = 28 x 28)
constexpr int kLdX1 = 32 * kRT + 1;     // Xs[k][row]: the transposed store is conflict-free
constexpr int kLdW1 = kHidPad + 1;      // Ws[k][unit]
constexpr int kKc3 = 112;               // fc1 weight-gradient column chunk (784 = 7 x 112): 16 lanes x 7 columns
constexpr int kLdA = kHid + 1;          // A / delta1 rows
constexpr float kLr = 0.1f, kWeightDecay = 1e-4f;                    // backdoor.py:134

// shared memory, in floats
constexpr int kSmA = kMaxBatch * kLdA;                  // relu(fc1) rows, then delta1 rows
constexpr int kSmP = kMaxBatch * kOut;                  // logits, then delta2 rows
constexpr int kSmW2 = kOut * kHid + 16;                 // fc2.weight, fc2.bias
constexpr int kSmFwd = kKc1 * kLdX1 + kKc1 * kLdW1;
constexpr int kSmX3 = kMaxBatch * kKc3;
constexpr int kSmScratch = kSmFwd > kSmX3 ? kSmFwd : kSmX3;
constexpr size_t kSmemBytes = sizeof(float) * (kSmA + kSmP + kSmW2 + kSmScratch + kMaxBatch) + sizeof(int) * kMaxBatch;

struct Smem {
  float* A; float* P; float* W2; float* b2; float* scratch; float* nll; int* label;
};

__device__ __forceinline__ Smem carve(float* base) {
  Smem s;
  s.A = base; s.P = s.A + kSmA; s.W2 = s.P + kSmP; s.b2 = s.W2 + kOut * kHid; s.scratch = s.W2 + kSmW2;
  s.nll = s.scratch + kSmScratch; s.label = reinterpret_cast<int*>(s.nll + kMaxBatch);
  return s;
}

// torch.relu: NaN stays NaN (fmaxf would turn it into 0).
__device__ __forceinline__ float relu(float v) { return v > 0.f || v != v ? v : 0.f; }

// The forward pass of rows x[0..mb) (784 contiguous floats each) at the parameters w, to the logits in s.P:
// A[i][j] = relu(sum_k x_i[k] W1[j][k] + b1[j]) (k in order, then the bias) and P[i][c] = sum_j A[i][j] W2[c][j] + b2[c]
// (j in order).  Thread (tx, ty) owns hidden units tx + 16c and rows ty + 32r.  Also stages fc2 and the labels ys[0..mb).
// w may be the vector being trained: it is read through ordinary loads only.  Starts and ends at a barrier.
__device__ void forward(const float* __restrict__ x, const int64_t* __restrict__ ys, const float* w, int mb,
                        const Smem& s) {
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  for (int idx = t; idx < kOut * kHid + kOut; idx += kThreads)
    (idx < kOut * kHid ? s.W2[idx] : s.b2[idx - kOut * kHid]) = w[kOffW2 + idx];
  for (int i = t; i < mb; i += kThreads) s.label[i] = static_cast<int>(ys[i]);
  float* Xs = s.scratch;
  float* Ws = s.scratch + kKc1 * kLdX1;
  float acc[kRT][7];
#pragma unroll
  for (int r = 0; r < kRT; ++r)
#pragma unroll
    for (int c = 0; c < 7; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < kIn; k0 += kKc1) {
    __syncthreads();
    for (int idx = t; idx < 32 * kRT * kKc1; idx += kThreads) {
      const int i = idx / kKc1, kk = idx % kKc1;
      Xs[kk * kLdX1 + i] = i < mb ? x[int64_t(i) * kIn + k0 + kk] : 0.f;
    }
    for (int idx = t; idx < kHidPad * kKc1; idx += kThreads) {
      const int j = idx / kKc1, kk = idx % kKc1;
      Ws[kk * kLdW1 + j] = j < kHid ? w[j * kIn + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kKc1; ++kk) {
      float xv[kRT], wv[7];
#pragma unroll
      for (int r = 0; r < kRT; ++r) xv[r] = Xs[kk * kLdX1 + ty + 32 * r];
#pragma unroll
      for (int c = 0; c < 7; ++c) wv[c] = Ws[kk * kLdW1 + tx + 16 * c];
#pragma unroll
      for (int r = 0; r < kRT; ++r)
#pragma unroll
        for (int c = 0; c < 7; ++c) acc[r][c] = fmaf(xv[r], wv[c], acc[r][c]);
    }
  }
#pragma unroll
  for (int c = 0; c < 7; ++c) {
    const int j = tx + 16 * c;
    if (j >= kHid) continue;
    const float bj = w[kOffB1 + j];
#pragma unroll
    for (int r = 0; r < kRT; ++r) {
      const int i = ty + 32 * r;
      if (i < mb) s.A[i * kLdA + j] = relu(acc[r][c] + bj);
    }
  }
  __syncthreads();
  for (int idx = t; idx < mb * kOut; idx += kThreads) {
    const int i = idx / kOut, c = idx % kOut;
    float z = 0.f;
    for (int j = 0; j < kHid; ++j) z = fmaf(s.A[i * kLdA + j], s.W2[c * kHid + j], z);
    s.P[i * kOut + c] = z + s.b2[c];
  }
  __syncthreads();
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

// Row i's NLL (-logp[label]; NaN for a label outside 0..9) and whether torch's out.max(1)[1] is the label (the first
// NaN, else the first maximum).  delta: P[i] <- (softmax - onehot) / mb, NLLLoss(mean) through log_softmax's backward.
__device__ __forceinline__ float row_head(const Smem& s, int i, int mb, bool delta, bool* hit) {
  float z[kOut], lp[kOut];
#pragma unroll
  for (int c = 0; c < kOut; ++c) z[c] = s.P[i * kOut + c];
  log_softmax_row(z, lp);
  int best = 0;
#pragma unroll
  for (int c = 1; c < kOut; ++c)
    if (lp[best] == lp[best] && (lp[c] != lp[c] || lp[c] > lp[best])) best = c;
  const int yi = s.label[i];
  *hit = best == yi;
  if (delta) {
    const float fmb = static_cast<float>(mb);
#pragma unroll
    for (int c = 0; c < kOut; ++c) s.P[i * kOut + c] = (expf(lp[c]) - (c == yi ? 1.f : 0.f)) / fmb;
  }
  return yi >= 0 && yi < kOut ? -lp[yi] : __int_as_float(0x7fc00000);
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
    forward(xs + int64_t(lo) * kIn, ys + lo, w, mb, s);
    bool hit = false;
    if (threadIdx.x < mb) s.nll[threadIdx.x] = row_head(s, threadIdx.x, mb, false, &hit);
    correct += __syncthreads_count(hit);
    if (threadIdx.x == 0) {
      float sum = 0.f;
      for (int i = 0; i < mb; ++i) sum += s.nll[i];
      total += static_cast<double>(sum / static_cast<float>(mb));
    }
  }
  *loss = total;
  return correct;
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

__global__ void __launch_bounds__(kThreads, 1)
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
  const Smem s = carve(smem);
  const float* xs = x + int64_t(set) * max_len * kIn;
  const int64_t* ys = y + int64_t(set) * max_len;
  const float* p0 = initial + int64_t(b) * kD;
  float* p = out + int64_t(b) * kD;
  // the output starts as initial; p0 - p0 is NaN where initial holds a NaN or an infinity (the first dist loss)
  bool bad = false;
  for (int c = t; c < kD; c += kThreads) {
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
      const float* xb = xs + int64_t(lo) * kIn;
      forward(xb, ys + lo, p, mb, s);
      bool hit, nan_row = false;
      if (t < mb) {
        const float l = row_head(s, t, mb, true, &hit);
        nan_row = l != l;
      }
      if (__syncthreads_or(nan_row)) {                                  // "Got nan loss"
        if (t == 0) status[b] = AFL_ERR_NAN_LOSS;
        return;
      }
      // fc2: dW2[c][j] = sum_i delta2[i][c] A[i][j], db2[c] = sum_i delta2[i][c] (i in order), kept until delta1 has
      // read the old fc2
      float g2[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int idx = t + q * kThreads;
        float acc = 0.f;
        if (idx < kOut * kHid) {
          const int c = idx / kHid, j = idx % kHid;
          for (int i = 0; i < mb; ++i) acc = fmaf(s.P[i * kOut + c], s.A[i * kLdA + j], acc);
        } else if (idx < kOut * kHid + kOut) {
          const int c = idx - kOut * kHid;
          for (int i = 0; i < mb; ++i) acc += s.P[i * kOut + c];
        }
        g2[q] = acc;
      }
      __syncthreads();
      // delta1 = (delta2 W2) * (A > 0), in place of A (threshold_backward: zero where the activation is <= 0)
      for (int idx = t; idx < mb * kHid; idx += kThreads) {
        const int i = idx / kHid, j = idx % kHid;
        float d = 0.f;
#pragma unroll
        for (int c = 0; c < kOut; ++c) d = fmaf(s.P[i * kOut + c], s.W2[c * kHid + j], d);
        s.A[i * kLdA + j] = s.A[i * kLdA + j] > 0.f ? d : 0.f;
      }
      bad = false;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int idx = t + q * kThreads;
        if (idx < kOut * kHid + kOut) {
          const int o = kOffW2 + idx;
          const float norm = idx < kOut * kHid ? 2.f / (kOut * kHid) : 2.f / kOut;
          p[o] = sgd(p[o], p0[o], g2[q], norm, alpha, dist, &bad);
        }
      }
      __syncthreads();
      if (t < kHid) {                                                   // fc1.bias: db1[j] = sum_i delta1[i][j]
        float acc = 0.f;
        for (int i = 0; i < mb; ++i) acc += s.A[i * kLdA + t];
        const int o = kOffB1 + t;
        p[o] = sgd(p[o], p0[o], acc, 2.f / kHid, alpha, dist, &bad);
      }
      // fc1.weight: dW1[j][k] = sum_i delta1[i][j] x_i[k], 112 columns at a time.  Thread (tx, ty) owns columns
      // tx + 16e and units ty + 32c; only ty < 4 has a fourth unit (96..99).
      const int tx = t & 15, ty = t >> 4;
      float* Xc = s.scratch;
      for (int k0 = 0; k0 < kIn; k0 += kKc3) {
        for (int idx = t; idx < mb * kKc3; idx += kThreads) {
          const int i = idx / kKc3, kk = idx % kKc3;
          Xc[idx] = xb[int64_t(i) * kIn + k0 + kk];
        }
        __syncthreads();
        float acc[4][7];
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int e2 = 0; e2 < 7; ++e2) acc[c][e2] = 0.f;
        const bool c3 = ty + 96 < kHid;
        for (int i = 0; i < mb; ++i) {
          float xv[7], dv[4];
#pragma unroll
          for (int e2 = 0; e2 < 7; ++e2) xv[e2] = Xc[i * kKc3 + tx + 16 * e2];
#pragma unroll
          for (int c = 0; c < 3; ++c) dv[c] = s.A[i * kLdA + ty + 32 * c];
          dv[3] = c3 ? s.A[i * kLdA + ty + 96] : 0.f;
#pragma unroll
          for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int e2 = 0; e2 < 7; ++e2) acc[c][e2] = fmaf(dv[c], xv[e2], acc[c][e2]);
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = ty + 32 * c;
          if (j >= kHid) continue;
#pragma unroll
          for (int e2 = 0; e2 < 7; ++e2) {
            const int o = j * kIn + k0 + tx + 16 * e2;
            p[o] = sgd(p[o], p0[o], acc[c][e2], 2.f / (kHid * kIn), alpha, dist, &bad);
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
__global__ void __launch_bounds__(kThreads, 1)
backdoor_test_kernel(const float* __restrict__ weights, int batch, const float* __restrict__ x,
                     const int64_t* __restrict__ y, int n_sets, int max_len, const int* __restrict__ set_len,
                     const int* __restrict__ data_index, int m, const int* __restrict__ slot, int n_slots,
                     double* __restrict__ loss_sum, int* __restrict__ correct) {
  const int b = blockIdx.x;
  const int set = data_index[b], sl = *slot;
  const int len = set >= 0 && set < n_sets ? set_len[set] : 0;
  if (len < 1 || len > max_len || sl < 0 || sl >= n_slots) return;
  extern __shared__ float smem[];
  const Smem s = carve(smem);
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

// The checks both calls share: pointers are checked by the callers.
static int check_common(const char* who, int batch, int64_t d, int n_sets, int max_len, int m) {
  if (batch < 1 || n_sets < 1 || max_len < 1 || m < 1) {
    set_error("%s: batch, n_sets, max_len and m must be >= 1 (got %d, %d, %d, %d)", who, batch, n_sets, max_len, m);
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

}  // namespace backdoor
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
  if (int rc = backdoor::check_common(who, batch, d, n_sets, max_len, m)) return rc;
  if (mal_epochs < 0 || alpha != alpha) {
    set_error("%s: mal_epochs must be >= 0 and alpha a number (got %d, %g)", who, mal_epochs, alpha);
    return AFL_ERR_BAD_ARG;
  }
  const uintptr_t span = static_cast<uintptr_t>(batch) * backdoor::kD * sizeof(float);
  const uintptr_t a = reinterpret_cast<uintptr_t>(initial), o = reinterpret_cast<uintptr_t>(out);
  if (a < o + span && o < a + span) { set_error("%s: out overlaps initial", who); return AFL_ERR_BAD_ARG; }
  AFL_CUDA(ensure_dyn_smem(backdoor::backdoor_train_kernel, static_cast<int>(backdoor::kSmemBytes),
                           backdoor::smem_done_train));
  ProfScope ps("backdoor_train", static_cast<cudaStream_t>(stream));
  backdoor::backdoor_train_kernel<<<batch, backdoor::kThreads, backdoor::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
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
  if (int rc = backdoor::check_common(who, batch, d, n_sets, max_len, m)) return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  AFL_CUDA(ensure_dyn_smem(backdoor::backdoor_test_kernel, static_cast<int>(backdoor::kSmemBytes),
                           backdoor::smem_done_test));
  backdoor::backdoor_test_kernel<<<batch, backdoor::kThreads, backdoor::kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
      weights, batch, x, y, n_sets, max_len, set_len, data_index, m, slot_index, n_slots, loss_sum, correct);
  AFL_LAUNCH_CHECK("backdoor_test_kernel");
  return AFL_OK;
}

}  // extern "C"
