// MnistNet device code shared by the client-gradient and evaluation kernels (client_grad.cu) and the backdoor
// attacker's trainer and backdoor test (backdoor_train.cu): the layout, the block geometry, the shared-memory carve and
// the passes both restate (DESIGN 2.6).
//
// The net is harness.MnistNet (data_sets.py:13-24): log_softmax(fc2(relu(fc1(x)))), fc1 [100, 784], fc2 [10, 100],
// flattened in ParamLayout order (fc1.weight, fc1.bias, fc2.weight, fc2.bias; D = 79,510).
#pragma once
#include "train_common.cuh"

namespace afl {
namespace mnist {

constexpr int kIn = 784, kHid = 100, kOut = train::kClasses;
constexpr int64_t kD = int64_t(kHid) * kIn + kHid + kOut * kHid + kOut;        // 79,510
constexpr int kOffB1 = kHid * kIn, kOffW2 = kOffB1 + kHid, kOffB2 = kOffW2 + kOut * kHid;
constexpr int kHidPad = 112;            // forward: 16 unit lanes x 7 hidden units
constexpr int kLdW1 = kHidPad + 1;      // Ws[k][unit]
constexpr int kLdA = kHid + 1;          // A / delta1 rows

// A kernel family's block geometry: kThreads threads, minibatches of up to kRows rows, forward k-chunks of kKc1 columns.
// The forward gives thread (tx, ty) = (t % 16, t / 16) hidden units tx + 16c and rows ty + kRowLanes r; the fc1
// weight gradient gives it columns t % kColLanes + kColLanes e (7 of them, a kKc3-column chunk) and units
// t / kColLanes + 32c.
template <int kThreads_, int kRows_, int kKc1_>
struct Geometry {
  static constexpr int kThreads = kThreads_, kRows = kRows_, kKc1 = kKc1_;
  static constexpr int kRowLanes = kThreads / 16;
  static constexpr int kLdX1 = (kRows + kRowLanes - 1) / kRowLanes * kRowLanes + 1;   // Xs[k][row]: conflict-free
  static constexpr int kColLanes = kThreads / 32;
  static constexpr int kKc3 = 7 * kColLanes;
  static_assert(kIn % kKc1 == 0 && kIn % kKc3 == 0, "the chunks tile fc1's 784 columns");
  // shared memory, in floats: relu(fc1) rows, then delta1 rows; logits, then delta2 rows; fc2.weight; the forward's
  // k-chunks or the weight gradient's column chunk; then the minibatch's labels
  static constexpr int kSmA = kRows * kLdA, kSmP = kRows * kOut, kSmW2 = kOut * kHid;
  static constexpr int kSmFwd = kKc1 * kLdX1 + kKc1 * kLdW1, kSmX3 = kRows * kKc3;
  static constexpr int kSmScratch = kSmFwd > kSmX3 ? kSmFwd : kSmX3;
  static constexpr size_t kSmemBytes = sizeof(float) * (kSmA + kSmP + kSmW2 + kSmScratch) + sizeof(int) * kRows;
};

struct Smem {
  float* A; float* P; float* W2; float* scratch; int* label;
};

template <class G>
__device__ __forceinline__ Smem carve(float* base) {
  Smem s;
  s.A = base; s.P = s.A + G::kSmA; s.W2 = s.P + G::kSmP; s.scratch = s.W2 + G::kSmW2;
  s.label = reinterpret_cast<int*>(s.scratch + G::kSmScratch);
  return s;
}

template <class G>
__device__ __forceinline__ void stage_w2(const float* w, const Smem& s) {
  for (int idx = threadIdx.x; idx < kOut * kHid; idx += G::kThreads) s.W2[idx] = w[kOffW2 + idx];
}

// Forward through relu(fc1): A[i][j] = relu(sum_k x_i[k] W1[j][k] + b1[j]) for i < mb <= kRowLanes RT, j < 100, with
// minibatch row i at x0 + i pitch; each sum runs k = 0..783 in order, then adds the bias.  Leaves the last chunk's
// barrier behind it.
template <class G, int RT>
__device__ __forceinline__ void forward_hidden(const float* __restrict__ x0, int64_t pitch, const float* w, int mb,
                                               const Smem& s) {
  constexpr int kKc1 = G::kKc1, kLdX1 = G::kLdX1;
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  float* Xs = s.scratch;
  float* Ws = s.scratch + kKc1 * kLdX1;
  float acc[RT][7];
#pragma unroll
  for (int r = 0; r < RT; ++r)
#pragma unroll
    for (int c = 0; c < 7; ++c) acc[r][c] = 0.f;
  for (int k0 = 0; k0 < kIn; k0 += kKc1) {
    for (int idx = t; idx < G::kRowLanes * RT * kKc1; idx += G::kThreads) {
      const int i = idx / kKc1, kk = idx % kKc1;
      Xs[kk * kLdX1 + i] = i < mb ? x0[i * pitch + k0 + kk] : 0.f;
    }
    for (int idx = t; idx < kHidPad * kKc1; idx += G::kThreads) {
      const int j = idx / kKc1, kk = idx % kKc1;
      Ws[kk * kLdW1 + j] = j < kHid ? w[j * kIn + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int kk = 0; kk < kKc1; ++kk) {
      float xv[RT], wv[7];
#pragma unroll
      for (int r = 0; r < RT; ++r) xv[r] = Xs[kk * kLdX1 + ty + G::kRowLanes * r];
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
      const int i = ty + G::kRowLanes * r;
      if (i < mb) s.A[i * kLdA + j] = train::relu(acc[r][c] + bj);
    }
  }
}

// logits P[i][c] = sum_j A[i][j] W2[c][j] (j in order) + b2[c]; W2 is staged into s.W2 first.
template <class G>
__device__ __forceinline__ void forward_logits(const float* w, int mb, const Smem& s) {
  for (int idx = threadIdx.x; idx < mb * kOut; idx += G::kThreads) {
    const int i = idx / kOut, c = idx % kOut;
    float z = 0.f;
    for (int j = 0; j < kHid; ++j) z = fmaf(s.A[i * kLdA + j], s.W2[c * kHid + j], z);
    s.P[i * kOut + c] = z + w[kOffB2 + c];
  }
}

// fc2's gradient: dW2[c][j] = sum_i delta2[i][c] A[i][j] for idx = c kHid + j, and db2[c] = sum_i delta2[i][c], i in
// order.
__device__ __forceinline__ float fc2_weight_grad(int idx, int mb, const Smem& s) {
  const int c = idx / kHid, j = idx % kHid;
  float acc = 0.f;
  for (int i = 0; i < mb; ++i) acc = fmaf(s.P[i * kOut + c], s.A[i * kLdA + j], acc);
  return acc;
}
__device__ __forceinline__ float fc2_bias_grad(int c, int mb, const Smem& s) {
  float acc = 0.f;
  for (int i = 0; i < mb; ++i) acc += s.P[i * kOut + c];
  return acc;
}

// delta1 = delta2 W2 where A is not <= 0, in place of A (threshold_backward: zero where the ReLU output is <= 0, the
// gradient elsewhere, a NaN output included)
template <class G>
__device__ __forceinline__ void backward_hidden(int mb, const Smem& s) {
  for (int idx = threadIdx.x; idx < mb * kHid; idx += G::kThreads) {
    const int i = idx / kHid, j = idx % kHid;
    float d = 0.f;
#pragma unroll
    for (int c = 0; c < kOut; ++c) d = fmaf(s.P[i * kOut + c], s.W2[c * kHid + j], d);
    s.A[i * kLdA + j] = s.A[i * kLdA + j] <= 0.f ? 0.f : d;
  }
}

// fc1's weight gradient over columns k0 .. k0 + kKc3: acc[c][e] = dW1[j][k] = sum_i delta1[i][j] x_i[k] for unit
// j = t / kColLanes + 32c and column k = k0 + t % kColLanes + kColLanes e (only j < 100 is meaningful; the warps
// with no fourth unit skip it as a whole).  Stages the chunk in s.scratch; the caller consumes acc and then needs a
// barrier before the next chunk.
template <class G>
__device__ __forceinline__ void fc1_weight_grad(const float* __restrict__ x0, int64_t pitch, int k0, int mb,
                                                const Smem& s, float (&acc)[4][7]) {
  constexpr int kKc3 = G::kKc3;
  const int tx = threadIdx.x % G::kColLanes, ty = threadIdx.x / G::kColLanes;
  float* Xc = s.scratch;
  for (int idx = threadIdx.x; idx < mb * kKc3; idx += G::kThreads) {
    const int i = idx / kKc3, kk = idx % kKc3;
    Xc[idx] = x0[i * pitch + k0 + kk];
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int e = 0; e < 7; ++e) acc[c][e] = 0.f;
  const bool c3 = ty + 96 < kHid;
  for (int i = 0; i < mb; ++i) {
    float xv[7], dv[4];
#pragma unroll
    for (int e = 0; e < 7; ++e) xv[e] = Xc[i * kKc3 + tx + G::kColLanes * e];
#pragma unroll
    for (int c = 0; c < 3; ++c) dv[c] = s.A[i * kLdA + ty + 32 * c];
    dv[3] = c3 ? s.A[i * kLdA + ty + 96] : 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int e = 0; e < 7; ++e) acc[c][e] = fmaf(dv[c], xv[e], acc[c][e]);
  }
}

}  // namespace mnist
}  // namespace afl
