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
// gradient to that index alone.
#include "afl_common.cuh"

namespace afl {
namespace cifar {

constexpr int kImg = 3 * 32 * 32;                       // one NCHW image, flattened
constexpr int kC1 = 16, kC2 = 64, kH1 = 384, kH2 = 192, kOut = 10;
constexpr int kOffW1c = 0, kOffB1c = 432, kOffW2c = 448, kOffB2c = 16'832, kOffW1 = 16'896, kOffB1 = 41'472;
constexpr int kOffW2 = 41'856, kOffB2 = 115'584, kOffW3 = 115'776, kOffB3 = 117'696;
constexpr int64_t kD = 117'706;
constexpr int kThreads = 256;
constexpr int kMaxBatch = 128;
constexpr int kS = 16;                                  // minibatch rows per chunk
constexpr int kCells = 49;                              // pool1's 7x7 corner
constexpr int kP1 = kC1 * kCells;                       // 784 pool1 values per row
constexpr int kLdP1 = kP1 + 1;                          // odd: rows s of a warp hit distinct banks

// shared memory, in floats (the byte arrays at the end)
constexpr int kSmW1c = kOffW2c;                         // conv1 weights and bias
constexpr int kSmP1 = kS * kLdP1;                       // pool1 values, then their gradients
constexpr int kSmH = kS * kC2;                          // pool2 values (fc1 input), then their gradients
constexpr int kSmA1 = kS * kH1;                         // relu(fc1), then delta1
constexpr int kSmA2 = kS * kH2;                         // relu(fc2), then delta2
constexpr int kSmZ = kS * kOut;                         // logits, then delta3
constexpr int kSmF = kSmW1c + kSmP1 + kSmH + kSmA1 + kSmA2 + kSmZ + 2 * kMaxBatch;   // + per-row NLL and hit
constexpr size_t kSmemBytes = sizeof(float) * kSmF + sizeof(int) * 2 * kMaxBatch + kS * kP1 + kS * kC2;

struct Smem {
  float* w1c; float* P1; float* H; float* A1; float* A2; float* Z; float* nll; float* hit;
  int* row; int* label; unsigned char* I1; unsigned char* I2;
};

__device__ __forceinline__ Smem carve(float* base) {
  Smem s;
  s.w1c = base; s.P1 = s.w1c + kSmW1c; s.H = s.P1 + kSmP1; s.A1 = s.H + kSmH; s.A2 = s.A1 + kSmA1;
  s.Z = s.A2 + kSmA2; s.nll = s.Z + kSmZ; s.hit = s.nll + kMaxBatch;
  s.row = reinterpret_cast<int*>(s.hit + kMaxBatch); s.label = s.row + kMaxBatch;
  s.I1 = reinterpret_cast<unsigned char*>(s.label + kMaxBatch); s.I2 = s.I1 + kS * kP1;
  return s;
}

// torch.relu: NaN stays NaN (fmaxf would turn it into 0).  (client_grad.cu and backdoor_train.cu hold the same.)
__device__ __forceinline__ float relu(float v) { return v > 0.f || v != v ? v : 0.f; }

// torch's max_pool2d window step: a larger value or a NaN takes the index, so ties keep the first maximum.
__device__ __forceinline__ void pool_step(float v, int k, float& mx, int& mi) {
  if (v > mx || v != v) { mx = v; mi = k; }
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

// Client u's minibatch at epoch e: client_grad.cu's batch_start (harness.Client.step's cycling position).
__device__ __forceinline__ int batch_start(int n_train, int n, int u, int m, int e, int* mb) {
  const int L = (n_train - u + n - 1) / n;
  const int q = (L + m - 1) / m;
  int k = e % q;
  if (k < 0) k += q;
  const int lo = k * m;
  *mb = min(lo + m, L) - lo;
  return lo;
}

// The forward pass of rows row[c0 .. c0 + mc) into the chunk buffers: P1/I1, H/I2, A1, A2 and the logits Z.
// s.w1c must hold conv1's weights and bias.
__device__ void forward_chunk(const float* __restrict__ xs, const float* __restrict__ w, int c0, int mc,
                              const Smem& s) {
  const int t = threadIdx.x;
  // conv1 + relu + pool1 over the 7x7 corner: item (row, cell, channel), channel fastest (16 channels share a patch).
  // Each conv1 output sums ci, ky, kx in order, then adds the bias.
  for (int idx = t; idx < mc * kP1; idx += kThreads) {
    const int i = idx / kP1, r = idx % kP1, cell = r / kC1, c = r % kC1, py = cell / 7, px = cell % 7;
    const float* xp = xs + int64_t(s.row[c0 + i]) * kImg + (3 * py) * 32 + 3 * px;
    float acc[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) acc[q] = 0.f;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
      float p[5][5];
#pragma unroll
      for (int a = 0; a < 5; ++a)
#pragma unroll
        for (int b = 0; b < 5; ++b) p[a][b] = __ldg(xp + ci * 1024 + a * 32 + b);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float wv = s.w1c[c * 27 + ci * 9 + ky * 3 + kx];
#pragma unroll
          for (int ay = 0; ay < 3; ++ay)
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) acc[ay * 3 + ax] = fmaf(wv, p[ay + ky][ax + kx], acc[ay * 3 + ax]);
        }
    }
    const float bc = s.w1c[kOffB1c + c];
    float mx = -INFINITY;
    int mi = 0;
#pragma unroll
    for (int q = 0; q < 9; ++q) pool_step(relu(acc[q] + bc), q, mx, mi);
    s.P1[i * kLdP1 + c * kCells + cell] = mx;
    s.I1[i * kP1 + c * kCells + cell] = static_cast<unsigned char>(mi);
  }
  __syncthreads();
  // conv2 + relu + pool2 over conv2's 4x4 corner: item (channel, row), row fastest.  Each output sums ci, ky, kx in
  // order, then adds the bias.
  for (int idx = t; idx < mc * kC2; idx += kThreads) {
    const int co = idx / mc, i = idx % mc;
    const float* wc = w + kOffW2c + co * 256;
    const float* pp = s.P1 + i * kLdP1;
    float acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = 0.f;
#pragma unroll 1
    for (int ci = 0; ci < kC1; ++ci) {
      float p[7][7];
#pragma unroll
      for (int a = 0; a < 7; ++a)
#pragma unroll
        for (int b = 0; b < 7; ++b) p[a][b] = pp[ci * kCells + a * 7 + b];
#pragma unroll
      for (int ky = 0; ky < 4; ++ky)
#pragma unroll
        for (int kx = 0; kx < 4; ++kx) {
          const float wv = __ldg(wc + ci * 16 + ky * 4 + kx);
#pragma unroll
          for (int oy = 0; oy < 4; ++oy)
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) acc[oy * 4 + ox] = fmaf(wv, p[oy + ky][ox + kx], acc[oy * 4 + ox]);
        }
    }
    const float bc = __ldg(w + kOffB2c + co);
    float mx = -INFINITY;
    int mi = 0;
#pragma unroll
    for (int q = 0; q < 16; ++q) pool_step(relu(acc[q] + bc), q, mx, mi);
    s.H[i * kC2 + co] = mx;
    s.I2[i * kC2 + co] = static_cast<unsigned char>(mi);
  }
  __syncthreads();
  // fc1: A1[i][j] = relu(sum_k H[i][k] W1[j][k] + b1[j]), k in order
  for (int j = t; j < kH1; j += kThreads) {
    float acc[kS];
#pragma unroll
    for (int i = 0; i < kS; ++i) acc[i] = 0.f;
    const float* wr = w + kOffW1 + j * kC2;
#pragma unroll 4
    for (int k = 0; k < kC2; ++k) {
      const float wv = __ldg(wr + k);
#pragma unroll
      for (int i = 0; i < kS; ++i) acc[i] = fmaf(s.H[i * kC2 + k], wv, acc[i]);
    }
    const float bj = __ldg(w + kOffB1 + j);
#pragma unroll
    for (int i = 0; i < kS; ++i)
      if (i < mc) s.A1[i * kH1 + j] = relu(acc[i] + bj);
  }
  __syncthreads();
  // fc2: A2[i][j] = relu(sum_k A1[i][k] W2[j][k] + b2[j]), k in order; W2 comes from L2, shared by a problem's clients
  for (int j = t; j < kH2; j += kThreads) {
    float acc[kS];
#pragma unroll
    for (int i = 0; i < kS; ++i) acc[i] = 0.f;
    const float* wr = w + kOffW2 + j * kH1;
#pragma unroll 4
    for (int k = 0; k < kH1; ++k) {
      const float wv = __ldg(wr + k);
#pragma unroll
      for (int i = 0; i < kS; ++i) acc[i] = fmaf(s.A1[i * kH1 + k], wv, acc[i]);
    }
    const float bj = __ldg(w + kOffB2 + j);
#pragma unroll
    for (int i = 0; i < kS; ++i)
      if (i < mc) s.A2[i * kH2 + j] = relu(acc[i] + bj);
  }
  __syncthreads();
  // fc3: Z[i][c] = sum_j A2[i][j] W3[c][j] (j in order) + b3[c]
  for (int idx = t; idx < mc * kOut; idx += kThreads) {
    const int i = idx / kOut, c = idx % kOut;
    float z = 0.f;
    for (int j = 0; j < kH2; ++j) z = fmaf(s.A2[i * kH2 + j], __ldg(w + kOffW3 + c * kH2 + j), z);
    s.Z[idx] = z + __ldg(w + kOffB3 + c);
  }
  __syncthreads();
}

// The backward pass of the chunk (rows c0 .. c0 + mc of an mb-row minibatch): adds its rows to every weight gradient
// in g (first: the chunk starts the sums).  Overwrites Z, A2, A1, H and P1 with their gradients.
__device__ void backward_chunk(const float* __restrict__ xs, const float* __restrict__ w, int c0, int mc, int mb,
                               bool first, const Smem& s, float* __restrict__ g) {
  const int t = threadIdx.x;
  // delta3 = (softmax - onehot) / mb: NLLLoss(mean) through log_softmax's backward
  const float fmb = static_cast<float>(mb);
  for (int i = t; i < mc; i += kThreads) {
    float z[kOut], lp[kOut];
#pragma unroll
    for (int c = 0; c < kOut; ++c) z[c] = s.Z[i * kOut + c];
    log_softmax_row(z, lp);
    const int yi = s.label[c0 + i];
#pragma unroll
    for (int c = 0; c < kOut; ++c) s.Z[i * kOut + c] = (expf(lp[c]) - (c == yi ? 1.f : 0.f)) / fmb;
  }
  __syncthreads();
  // fc3: dW3[c][j] += sum_i delta3[i][c] A2[i][j], db3[c] += sum_i delta3[i][c]
  for (int e = t; e < kOut * kH2 + kOut; e += kThreads) {
    if (e < kOut * kH2) {
      const int c = e / kH2, j = e % kH2;
      float acc = first ? 0.f : g[kOffW3 + e];
      for (int i = 0; i < mc; ++i) acc = fmaf(s.Z[i * kOut + c], s.A2[i * kH2 + j], acc);
      g[kOffW3 + e] = acc;
    } else {
      const int c = e - kOut * kH2;
      float acc = first ? 0.f : g[kOffB3 + c];
      for (int i = 0; i < mc; ++i) acc += s.Z[i * kOut + c];
      g[kOffB3 + c] = acc;
    }
  }
  __syncthreads();
  // delta2 = delta3 W3 where A2 is not <= 0 (threshold_backward), in place of A2
  for (int idx = t; idx < mc * kH2; idx += kThreads) {
    const int i = idx / kH2, j = idx % kH2;
    float d = 0.f;
#pragma unroll
    for (int c = 0; c < kOut; ++c) d = fmaf(s.Z[i * kOut + c], __ldg(w + kOffW3 + c * kH2 + j), d);
    s.A2[idx] = s.A2[idx] <= 0.f ? 0.f : d;
  }
  __syncthreads();
  // fc2: dW2[j][k] += sum_i delta2[i][j] A1[i][k] in 4 x 4 register tiles: warp wy owns units j = wy + 8 r, lane
  // owns columns k = lane + 32 q.  db2[j] += sum_i delta2[i][j].
  {
    const int lane = t & 31, wy = t >> 5;
    for (int r0 = 0; r0 < kH2 / 8; r0 += 4)
      for (int q0 = 0; q0 < kH1 / 32; q0 += 4) {
        float acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q)
            acc[r][q] = first ? 0.f : g[kOffW2 + (wy + 8 * (r0 + r)) * kH1 + lane + 32 * (q0 + q)];
        for (int i = 0; i < mc; ++i) {
          float dv[4], av[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) dv[r] = s.A2[i * kH2 + wy + 8 * (r0 + r)];
#pragma unroll
          for (int q = 0; q < 4; ++q) av[q] = s.A1[i * kH1 + lane + 32 * (q0 + q)];
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[r][q] = fmaf(dv[r], av[q], acc[r][q]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) g[kOffW2 + (wy + 8 * (r0 + r)) * kH1 + lane + 32 * (q0 + q)] = acc[r][q];
      }
    for (int j = t; j < kH2; j += kThreads) {
      float acc = first ? 0.f : g[kOffB2 + j];
      for (int i = 0; i < mc; ++i) acc += s.A2[i * kH2 + j];
      g[kOffB2 + j] = acc;
    }
  }
  __syncthreads();
  // delta1 = delta2 W2 (j in order) where A1 is not <= 0, in place of A1
  for (int k = t; k < kH1; k += kThreads) {
    float acc[kS];
#pragma unroll
    for (int i = 0; i < kS; ++i) acc[i] = 0.f;
#pragma unroll 4
    for (int j = 0; j < kH2; ++j) {
      const float wv = __ldg(w + kOffW2 + j * kH1 + k);
#pragma unroll
      for (int i = 0; i < kS; ++i) acc[i] = fmaf(s.A2[i * kH2 + j], wv, acc[i]);
    }
#pragma unroll
    for (int i = 0; i < kS; ++i)
      if (i < mc) s.A1[i * kH1 + k] = s.A1[i * kH1 + k] <= 0.f ? 0.f : acc[i];
  }
  __syncthreads();
  // fc1: dW1[j][k] += sum_i delta1[i][j] H[i][k]: thread (k = t % 64, jg = t / 64) owns units j = jg + 4 r.
  // db1[j] += sum_i delta1[i][j].
  {
    const int k = t & 63, jg = t >> 6;
    for (int r0 = 0; r0 < kH1 / 4; r0 += 4) {
      float acc[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[r] = first ? 0.f : g[kOffW1 + (jg + 4 * (r0 + r)) * kC2 + k];
      for (int i = 0; i < mc; ++i) {
        const float hv = s.H[i * kC2 + k];
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[r] = fmaf(s.A1[i * kH1 + jg + 4 * (r0 + r)], hv, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) g[kOffW1 + (jg + 4 * (r0 + r)) * kC2 + k] = acc[r];
    }
    for (int j = t; j < kH1; j += kThreads) {
      float acc = first ? 0.f : g[kOffB1 + j];
      for (int i = 0; i < mc; ++i) acc += s.A1[i * kH1 + j];
      g[kOffB1 + j] = acc;
    }
  }
  __syncthreads();
  // the gradient at conv2's pool2 index: dH = delta1 W1 (j in order), zero where the pooled relu output H is <= 0;
  // in place of H
  for (int idx = t; idx < mc * kC2; idx += kThreads) {
    const int i = idx / kC2, k = idx % kC2;
    float d = 0.f;
    for (int j = 0; j < kH1; ++j) d = fmaf(s.A1[i * kH1 + j], __ldg(w + kOffW1 + j * kC2 + k), d);
    s.H[idx] = s.H[idx] <= 0.f ? 0.f : d;
  }
  __syncthreads();
  // conv2: dWc2[co][ci][ky][kx] += sum_i dH[i][co] P1[i][ci][oy + ky][ox + kx] at row i's pool2 index (oy, ox) of
  // channel co; dbc2[co] += sum_i dH[i][co].  Thread t owns (ci, ky, kx) = (t / 16, t / 4 % 4, t % 4) of every co.
  {
    const int ci = t >> 4, ky = (t >> 2) & 3, kx = t & 3;
    for (int co = 0; co < kC2; ++co) {
      float acc = first ? 0.f : g[kOffW2c + co * 256 + t];
      for (int i = 0; i < mc; ++i) {
        const int q = s.I2[i * kC2 + co];
        acc = fmaf(s.H[i * kC2 + co], s.P1[i * kLdP1 + ci * kCells + ((q >> 2) + ky) * 7 + (q & 3) + kx], acc);
      }
      g[kOffW2c + co * 256 + t] = acc;
    }
    if (t < kC2) {
      float acc = first ? 0.f : g[kOffB2c + t];
      for (int i = 0; i < mc; ++i) acc += s.H[i * kC2 + t];
      g[kOffB2c + t] = acc;
    }
  }
  __syncthreads();
  // pool1's gradient: dP1[i][ci][y][x] = sum_co dH[i][co] Wc2[co][ci][y - oy][x - ox] over the channels whose pool2
  // window reads (y, x) (co in order), zero where the pooled relu output P1 is <= 0; in place of P1
  for (int idx = t; idx < mc * kP1; idx += kThreads) {
    const int i = idx / kP1, r = idx % kP1, ci = r / kCells, cell = r % kCells, y = cell / 7, x = cell % 7;
    float d = 0.f;
    for (int co = 0; co < kC2; ++co) {
      const int q = s.I2[i * kC2 + co];
      const int ky = y - (q >> 2), kx = x - (q & 3);
      if (ky >= 0 && ky < 4 && kx >= 0 && kx < 4)
        d = fmaf(s.H[i * kC2 + co], __ldg(w + kOffW2c + co * 256 + ci * 16 + ky * 4 + kx), d);
    }
    float& p = s.P1[i * kLdP1 + r];
    p = p <= 0.f ? 0.f : d;
  }
  __syncthreads();
  // conv1: dWc1[c][ci][ky][kx] += sum_i (sum_cell dP1[i][c][cell] x_i[ci][3 py + ay + ky][3 px + ax + kx]) at each
  // cell's pool1 index (ay, ax); dbc1[c] += sum_i sum_cell dP1[i][c][cell].  Cells in order, then rows in order.
  for (int e = t; e < kOffW2c; e += kThreads) {
    float acc = first ? 0.f : g[e];
    if (e < kOffB1c) {
      const int c = e / 27, ci = e % 27 / 9, ky = e % 9 / 3, kx = e % 3;
      for (int i = 0; i < mc; ++i) {
        const float* xp = xs + int64_t(s.row[c0 + i]) * kImg + ci * 1024 + ky * 32 + kx;
        float part = 0.f;
        for (int cell = 0; cell < kCells; ++cell) {
          const int q = s.I1[i * kP1 + c * kCells + cell], py = cell / 7, px = cell % 7;
          part = fmaf(s.P1[i * kLdP1 + c * kCells + cell], __ldg(xp + (3 * py + q / 3) * 32 + 3 * px + q % 3), part);
        }
        acc += part;
      }
    } else {
      const int c = e - kOffB1c;
      for (int i = 0; i < mc; ++i) {
        float part = 0.f;
        for (int cell = 0; cell < kCells; ++cell) part += s.P1[i * kLdP1 + c * kCells + cell];
        acc += part;
      }
    }
    g[e] = acc;
  }
  __syncthreads();
}

__device__ __forceinline__ void stage_conv1(const float* __restrict__ w, const Smem& s) {
  for (int idx = threadIdx.x; idx < kSmW1c; idx += kThreads) s.w1c[idx] = __ldg(w + kOffW1c + idx);
}

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
  const int lo = batch_start(n_train, n, u, m, *epoch, &mb);
  for (int i = threadIdx.x; i < mb; i += kThreads) {
    const int r = u + n * (lo + i);
    s.row[i] = r;
    s.label[i] = static_cast<int>(ys[r]);
  }
  stage_conv1(w, s);
  __syncthreads();
  float* g = G + int64_t(b) * batch_stride + int64_t(u) * ld;
  for (int c0 = 0; c0 < mb; c0 += kS) {
    const int mc = min(kS, mb - c0);
    forward_chunk(xs, w, c0, mc, s);
    backward_chunk(xs, w, c0, mc, mb, c0 == 0, s, g);
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
  stage_conv1(w, s);
  __syncthreads();
  for (int c0 = 0; c0 < mb; c0 += kS) {
    const int mc = min(kS, mb - c0);
    forward_chunk(xs, w, c0, mc, s);
    // per row: its NLL, and 1 when the argmax (first maximum) is the label
    for (int i = threadIdx.x; i < mc; i += kThreads) {
      float z[kOut], lp[kOut];
#pragma unroll
      for (int c = 0; c < kOut; ++c) z[c] = s.Z[i * kOut + c];
      log_softmax_row(z, lp);
      int best = 0;
#pragma unroll
      for (int c = 1; c < kOut; ++c) best = lp[c] > lp[best] ? c : best;
      const int yi = s.label[c0 + i];
      s.nll[c0 + i] = yi >= 0 && yi < kOut ? -lp[yi] : __int_as_float(0x7fc00000);   // a label outside 0..9: NaN
      s.hit[c0 + i] = best == yi ? 1.f : 0.f;
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

static int smem_done_grad[kMaxDevices];
static int smem_done_eval[kMaxDevices];

static int check_common(const char* who, int batch, int64_t d, int n_sets, int n_rows, int m) {
  if (batch < 1 || n_sets < 1 || n_rows < 1 || m < 1) {
    set_error("%s: batch, n_sets, the set size and m must be >= 1 (got %d, %d, %d, %d)", who, batch, n_sets, n_rows, m);
    return AFL_ERR_BAD_ARG;
  }
  if (d != kD) {
    set_error("%s: the Cifar10Net layout has D = %lld parameters (got %lld)", who, static_cast<long long>(kD),
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
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(client_grad_kernel, static_cast<int>(kSmemBytes), smem_done_grad));
  client_grad_kernel<<<dim3(n, batch), kThreads, kSmemBytes, st>>>(
      weights, x, y, n_sets, n_rows, set_len, data_index, rows, n, m, epoch, G, batch_stride, ld);
  AFL_LAUNCH_CHECK("cifar_client_grad_kernel");
  return AFL_OK;
}

static int64_t eval_batches(int n_test, int m) { return (int64_t(n_test) + m - 1) / m; }

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
  if (batch < 1 || n_test < 1 || m < 1) return 0;
  const size_t per = static_cast<size_t>(batch) * cifar::eval_batches(n_test, m);
  return align_up(per * sizeof(float), 256) + align_up(per * sizeof(int), 256);
}

int afl_cifar10_evaluate(const float* weights, int batch, int64_t d, const float* x, const int64_t* y, int n_sets,
                         int n_test, const int* data_index, int m, const int* slot_index, int n_slots, double* loss_sum,
                         int* correct, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "afl_cifar10_evaluate";
  if (!weights || !x || !y || !data_index || !slot_index || !loss_sum || !correct || !workspace) {
    set_error("%s: a pointer argument is NULL", who);
    return AFL_ERR_BAD_ARG;
  }
  if (int rc = cifar::check_common(who, batch, d, n_sets, n_test, m)) return rc;
  if (n_slots < 1) { set_error("%s: n_slots must be >= 1 (got %d)", who, n_slots); return AFL_ERR_BAD_ARG; }
  const size_t need = afl_cifar10_evaluate_workspace_bytes(batch, n_test, m);
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 256) {
    set_error("%s: workspace too small or misaligned (%zu < %zu)", who, workspace_bytes, need);
    return AFL_ERR_WORKSPACE;
  }
  const int64_t nb = cifar::eval_batches(n_test, m);
  if (nb > 65535) { set_error("%s: at most 65535 test batches (got %lld)", who, static_cast<long long>(nb)); return AFL_ERR_UNSUPPORTED; }
  float* batch_loss = static_cast<float*>(workspace);
  int* batch_correct = reinterpret_cast<int*>(static_cast<char*>(workspace) +
                                              align_up(static_cast<size_t>(batch) * nb * sizeof(float), 256));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  AFL_CUDA(ensure_dyn_smem(cifar::evaluate_kernel, static_cast<int>(cifar::kSmemBytes), cifar::smem_done_eval));
  cifar::evaluate_kernel<<<dim3(static_cast<unsigned>(nb), batch), cifar::kThreads, cifar::kSmemBytes, st>>>(
      weights, x, y, n_sets, n_test, data_index, m, batch_loss, batch_correct);
  AFL_LAUNCH_CHECK("cifar_evaluate_kernel");
  cifar::evaluate_finish_kernel<<<(batch + 127) / 128, 128, 0, st>>>(batch, static_cast<int>(nb), data_index, n_sets,
                                                                     batch_loss, batch_correct, slot_index, n_slots,
                                                                     loss_sum, correct);
  AFL_LAUNCH_CHECK("cifar_evaluate_finish_kernel");
  return AFL_OK;
}

}  // extern "C"
