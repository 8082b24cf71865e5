// Cifar10Net device code shared by the client-gradient and evaluation kernels (cifar_grad.cu) and the backdoor
// attacker's trainer and backdoor test (cifar_backdoor.cu): the layout, the shared-memory carve and one chunk's
// forward and backward pass (DESIGN 2.9).
#pragma once
#include "train_common.cuh"

namespace afl {
namespace cifar {

constexpr int kImg = 3 * 32 * 32;                       // one NCHW image, flattened
constexpr int kC1 = 16, kC2 = 64, kH1 = 384, kH2 = 192, kOut = train::kClasses;
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
constexpr int kSmChunk = kSmW1c + kSmP1 + kSmH + kSmA1 + kSmA2 + kSmZ;
// + per-row NLL and hit, row index and label for `rows` minibatch rows, then the chunk's pool1 and pool2 indices
constexpr size_t smem_bytes(int rows) {
  return sizeof(float) * (kSmChunk + 2 * rows) + sizeof(int) * 2 * rows + kS * kP1 + kS * kC2;
}
constexpr size_t kSmemBytes = smem_bytes(kMaxBatch);

struct Smem {
  float* w1c; float* P1; float* H; float* A1; float* A2; float* Z; float* nll; float* hit;
  int* row; int* label; unsigned char* I1; unsigned char* I2;
};

__device__ __forceinline__ Smem carve(float* base, int rows = kMaxBatch) {
  Smem s;
  s.w1c = base; s.P1 = s.w1c + kSmW1c; s.H = s.P1 + kSmP1; s.A1 = s.H + kSmH; s.A2 = s.A1 + kSmA1;
  s.Z = s.A2 + kSmA2; s.nll = s.Z + kSmZ; s.hit = s.nll + rows;
  s.row = reinterpret_cast<int*>(s.hit + rows); s.label = s.row + rows;
  s.I1 = reinterpret_cast<unsigned char*>(s.label + rows); s.I2 = s.I1 + kS * kP1;
  return s;
}

using train::ldw;
using train::relu;

// torch's max_pool2d window step: a larger value or a NaN takes the index, so ties keep the first maximum.
__device__ __forceinline__ void pool_step(float v, int k, float& mx, int& mi) {
  if (v > mx || v != v) { mx = v; mi = k; }
}

// The forward pass of rows row[c0 .. c0 + mc) into the chunk buffers: P1/I1, H/I2, A1, A2 and the logits Z.
// s.w1c must hold conv1's weights and bias.
template <bool kNc>
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
          const float wv = ldw<kNc>(wc + ci * 16 + ky * 4 + kx);
#pragma unroll
          for (int oy = 0; oy < 4; ++oy)
#pragma unroll
            for (int ox = 0; ox < 4; ++ox) acc[oy * 4 + ox] = fmaf(wv, p[oy + ky][ox + kx], acc[oy * 4 + ox]);
        }
    }
    const float bc = ldw<kNc>(w + kOffB2c + co);
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
      const float wv = ldw<kNc>(wr + k);
#pragma unroll
      for (int i = 0; i < kS; ++i) acc[i] = fmaf(s.H[i * kC2 + k], wv, acc[i]);
    }
    const float bj = ldw<kNc>(w + kOffB1 + j);
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
      const float wv = ldw<kNc>(wr + k);
#pragma unroll
      for (int i = 0; i < kS; ++i) acc[i] = fmaf(s.A1[i * kH1 + k], wv, acc[i]);
    }
    const float bj = ldw<kNc>(w + kOffB2 + j);
#pragma unroll
    for (int i = 0; i < kS; ++i)
      if (i < mc) s.A2[i * kH2 + j] = relu(acc[i] + bj);
  }
  __syncthreads();
  // fc3: Z[i][c] = sum_j A2[i][j] W3[c][j] (j in order) + b3[c]
  for (int idx = t; idx < mc * kOut; idx += kThreads) {
    const int i = idx / kOut, c = idx % kOut;
    float z = 0.f;
    for (int j = 0; j < kH2; ++j) z = fmaf(s.A2[i * kH2 + j], ldw<kNc>(w + kOffW3 + c * kH2 + j), z);
    s.Z[idx] = z + ldw<kNc>(w + kOffB3 + c);
  }
  __syncthreads();
}

// The backward pass of the chunk (rows c0 .. c0 + mc of an mb-row minibatch): adds its rows to every weight gradient
// in g (first: the chunk starts the sums).  Overwrites Z, A2, A1, H and P1 with their gradients.
template <bool kNc>
__device__ void backward_chunk(const float* __restrict__ xs, const float* __restrict__ w, int c0, int mc, int mb,
                               bool first, const Smem& s, float* __restrict__ g) {
  const int t = threadIdx.x;
  // delta3 = (softmax - onehot) / mb: NLLLoss(mean) through log_softmax's backward
  const float fmb = static_cast<float>(mb);
  for (int i = t; i < mc; i += kThreads) {
    float lp[kOut];
    train::log_softmax_row(s.Z + i * kOut, lp);
    train::row_delta(lp, s.label[c0 + i], fmb, s.Z + i * kOut);
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
    for (int c = 0; c < kOut; ++c) d = fmaf(s.Z[i * kOut + c], ldw<kNc>(w + kOffW3 + c * kH2 + j), d);
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
      const float wv = ldw<kNc>(w + kOffW2 + j * kH1 + k);
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
    for (int j = 0; j < kH1; ++j) d = fmaf(s.A1[i * kH1 + j], ldw<kNc>(w + kOffW1 + j * kC2 + k), d);
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
        d = fmaf(s.H[i * kC2 + co], ldw<kNc>(w + kOffW2c + co * 256 + ci * 16 + ky * 4 + kx), d);
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

template <bool kNc>
__device__ __forceinline__ void stage_conv1(const float* __restrict__ w, const Smem& s) {
  for (int idx = threadIdx.x; idx < kSmW1c; idx += kThreads) s.w1c[idx] = ldw<kNc>(w + kOffW1c + idx);
}

}  // namespace cifar
}  // namespace afl
