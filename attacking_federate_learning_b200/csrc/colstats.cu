// HBM-bound column kernels: plain mean (defences.py:13-14), the ALIE mu/sigma/perturb reduction
// (malicious.py:18-19,35), Krum's row gather, and the server momentum step (server.py:89-90).
// All of them stream the row-major [n, d] matrix once with 16-byte loads; a thread owns VEC adjacent
// columns and walks down the rows, so every warp-level load is one contiguous segment of a row.  mean and
// alie take a batch of same-shape problems in grid y (input at b * g_batch, outputs at b * out_batch).
#include <type_traits>

#include "afl_common.cuh"

namespace afl {
namespace colstats {

constexpr int kBlock = 256;
constexpr int kUnroll = 8;

template <int VEC> struct Pack { float v[VEC]; };

// One 16-bit element (low half of `b16`) of a bf16 or fp16 matrix as fp32 (exact).
template <typename T> __device__ __forceinline__ float half_bits_to_f32(uint32_t b16);
template <> __device__ __forceinline__ float half_bits_to_f32<__nv_bfloat16>(uint32_t b16) { return bf16_bits_to_f32(b16); }
template <> __device__ __forceinline__ float half_bits_to_f32<__half>(uint32_t b16) { return f16_bits_to_f32(b16); }

// Load VEC consecutive columns of one row as fp32.  VEC = 4 (fp32, 16 B) or 8 (bf16 / fp16, 16 B) or 1 (scalar).
template <typename T, int VEC>
__device__ __forceinline__ Pack<VEC> load_pack(const T* p);
template <> __device__ __forceinline__ Pack<4> load_pack<float, 4>(const float* p) {
  const float4 t = ldg_stream_f4(reinterpret_cast<const float4*>(p));
  return Pack<4>{{t.x, t.y, t.z, t.w}};
}
template <> __device__ __forceinline__ Pack<1> load_pack<float, 1>(const float* p) { return Pack<1>{{__ldg(p)}}; }
template <> __device__ __forceinline__ Pack<8> load_pack<__nv_bfloat16, 8>(const __nv_bfloat16* p) {
  const uint4 t = ldg_stream_u4(reinterpret_cast<const uint4*>(p));
  Pack<8> r;
  const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.v[2 * i] = bf16_bits_to_f32(w[i] & 0xFFFFu);
    r.v[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
  }
  return r;
}
template <> __device__ __forceinline__ Pack<1> load_pack<__nv_bfloat16, 1>(const __nv_bfloat16* p) {
  return Pack<1>{{__bfloat162float(*p)}};
}
template <> __device__ __forceinline__ Pack<8> load_pack<__half, 8>(const __half* p) {
  const uint4 t = ldg_stream_u4(reinterpret_cast<const uint4*>(p));
  Pack<8> r;
  const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r.v[2 * i] = f16_bits_to_f32(w[i] & 0xFFFFu);
    r.v[2 * i + 1] = f16_bits_to_f32(w[i] >> 16);
  }
  return r;
}
template <> __device__ __forceinline__ Pack<1> load_pack<__half, 1>(const __half* p) { return Pack<1>{{__half2float(*p)}}; }

// Coherent variants (no .nc, no L1 bypass hint): used when the kernel also WRITES the matrix it reads
// (ALIE writing the crafted vector back into the malicious rows it just reduced).
template <typename T, int VEC>
__device__ __forceinline__ Pack<VEC> load_pack_coherent(const T* p) {
  Pack<VEC> r;
  if constexpr (sizeof(T) == 4) {
    if constexpr (VEC == 4) {
      float4 t;
      asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(t.x), "=f"(t.y), "=f"(t.z), "=f"(t.w) : "l"(p) : "memory");
      r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
    } else {
      float t;
      asm volatile("ld.global.f32 %0, [%1];" : "=f"(t) : "l"(p) : "memory");
      r.v[0] = t;
    }
  } else {
    if constexpr (VEC == 8) {
      uint32_t w[4];
      asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "l"(p) : "memory");
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if constexpr (std::is_same<T, __half>::value) {
          r.v[2 * i] = f16_bits_to_f32(w[i] & 0xFFFFu); r.v[2 * i + 1] = f16_bits_to_f32(w[i] >> 16);
        } else {
          r.v[2 * i] = bf16_bits_to_f32(w[i] & 0xFFFFu); r.v[2 * i + 1] = __uint_as_float(w[i] & 0xFFFF0000u);
        }
      }
    } else {
      uint16_t t;
      asm volatile("ld.global.u16 %0, [%1];" : "=h"(t) : "l"(p) : "memory");
      r.v[0] = half_bits_to_f32<T>(t);
    }
  }
  return r;
}
template <typename T, int VEC, bool COHERENT>
__device__ __forceinline__ Pack<VEC> load_rows(const T* p) {
  if constexpr (COHERENT) return load_pack_coherent<T, VEC>(p);
  else return load_pack<T, VEC>(p);
}

// ---- mean: sequential fp32 row accumulation, then one IEEE division — the order NumPy uses for
// np.mean(axis=0) on a C-contiguous array, so fp32 results are bit-identical to the reference.
// kRows (a ragged batch): problem b averages its rows 0..each[b].tm.n_rows-1.
template <typename T, int VEC, bool kRows>
__global__ void __launch_bounds__(kBlock)
mean_kernel(const T* __restrict__ G, int n, int64_t d, int64_t ld, float* __restrict__ out, int64_t g_batch,
            int64_t out_batch, const ProblemParams* __restrict__ each) {
  const int64_t c0 = (static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x) * VEC;
  if (c0 >= d) return;
  if constexpr (kRows) n = each[blockIdx.y].tm.n_rows;
  G += blockIdx.y * g_batch;
  out += blockIdx.y * out_batch;
  float acc[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
  const T* p = G + c0;
  int r = 0;
  for (; r + kUnroll <= n; r += kUnroll) {
    Pack<VEC> t[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) t[u] = load_pack<T, VEC>(p + static_cast<int64_t>(r + u) * ld);
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[k] = __fadd_rn(acc[k], t[u].v[k]);
  }
  for (; r < n; ++r) {
    Pack<VEC> t = load_pack<T, VEC>(p + static_cast<int64_t>(r) * ld);
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = __fadd_rn(acc[k], t.v[k]);
  }
  const float fn = static_cast<float>(n);
#pragma unroll
  for (int k = 0; k < VEC; ++k)
    if (c0 + k < d) out[c0 + k] = __fdiv_rn(acc[k], fn);
}

// ---- ALIE: one pass, sum(x) and sum(x^2) per column in FLOAT64 (H100's FP64 pipe runs at half the FP32 rate: 3 FP64
// instructions per value hide under the HBM stream).  x*x is exact in float64 and the sums carry ~1e-16 relative error, so
// E[x^2] - E[x]^2 is accurate even when one client is orders of magnitude larger than the column's sigma (the
// round-1 version shifted by the first row in fp32 and lost ~1e-5 relative there).  sigma = sqrt(population
// variance); crafted = mu - z*sigma with the same two fp32 roundings as `grads_mean[:] -= num_std * grads_stdev[:]`.
// With a table (each != NULL) problem b uses its own f, z and write flag; f = 0 reads and writes no row and gives NaN
// statistics (the reference returns before computing any, malicious.py:11-12).  A column holding an inf has mu = +-inf
// (NaN with both signs) and, as np.var's inf - inf, sigma = NaN, so its crafted value is NaN.
// W: the element type of bcast, float (every existing caller) or T (alie_write16_kernel: a 16-bit matrix written in its
// own dtype, rounded to nearest even as torch's .to(dtype) does on the device).
template <typename W> __device__ __forceinline__ W from_f32(float x);
template <> __device__ __forceinline__ float from_f32<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
__device__ __forceinline__ uint32_t bits16(__nv_bfloat16 x) { return __bfloat16_as_ushort(x); }
__device__ __forceinline__ uint32_t bits16(__half x) { return __half_as_ushort(x); }

template <typename T, int VEC, bool COHERENT, typename W>
__device__ __forceinline__ void alie_body(const T* G, int f, int64_t d, int64_t ld, float z, float* __restrict__ mu_out,
                                          float* __restrict__ sigma_out, float* __restrict__ crafted_out, W* bcast,
                                          int64_t bcast_ld, int64_t g_batch, int64_t out_batch, int64_t bcast_batch,
                                          const ProblemParams* __restrict__ each) {
  const int64_t c0 = (static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x) * VEC;
  if (c0 >= d) return;
  if (each) {
    const ProblemParams& q = each[blockIdx.y];
    f = q.f; z = q.z;
    if (!q.write) bcast = nullptr;
  }
  G += blockIdx.y * g_batch;
  const T* p = G + c0;
  double s1[VEC], s2[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) { s1[k] = 0.0; s2[k] = 0.0; }
  int r = 0;
  for (; r + kUnroll <= f; r += kUnroll) {
    Pack<VEC> t[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) t[u] = load_rows<T, VEC, COHERENT>(p + static_cast<int64_t>(r + u) * ld);
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        const double x = static_cast<double>(t[u].v[k]);
        s1[k] += x;
        s2[k] = fma(x, x, s2[k]);
      }
  }
  for (; r < f; ++r) {
    Pack<VEC> t = load_rows<T, VEC, COHERENT>(p + static_cast<int64_t>(r) * ld);
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      const double x = static_cast<double>(t.v[k]);
      s1[k] += x;
      s2[k] = fma(x, x, s2[k]);
    }
  }
  const double inv = 1.0 / static_cast<double>(f);
  const int64_t o = blockIdx.y * out_batch + c0;         // this thread's first output element
  float crafted[VEC];
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const double m = s1[k] * inv;
    double var = fma(-m, m, s2[k] * inv);
    var = var < 0.0 ? 0.0 : var;                    // NaN stays NaN: f = 0, or an inf or NaN in the column (np.var)
    const float mu = static_cast<float>(m);
    const float sigma = static_cast<float>(sqrt(var));
    crafted[k] = __fsub_rn(mu, __fmul_rn(z, sigma));
    if (c0 + k < d) {
      if (sigma_out) sigma_out[o + k] = sigma;
      if (mu_out && mu_out != crafted_out) mu_out[o + k] = mu;
      if (crafted_out) crafted_out[o + k] = crafted[k];
    }
  }
  if (bcast) {
    bcast += blockIdx.y * bcast_batch;
    // server.py:82-83 copies the one aliased array into every malicious row: f row segments of VEC floats,
    // written as 16-byte stores when the destination allows it (all of this thread's reads are done)
    constexpr int kPer16 = 16 / sizeof(W);               // elements of one 16-byte store
    const bool v16 = (VEC % kPer16 == 0) && (c0 + VEC <= d) && (bcast_ld % kPer16 == 0) && ((reinterpret_cast<uintptr_t>(bcast) & 15) == 0);
    for (int rr = 0; rr < f; ++rr) {
      W* dst = bcast + static_cast<int64_t>(rr) * bcast_ld + c0;
      if constexpr (sizeof(W) == 4) {
        if (v16) {
#pragma unroll
          for (int k = 0; k + 4 <= VEC; k += 4) *reinterpret_cast<float4*>(dst + k) = make_float4(crafted[k], crafted[k + 1], crafted[k + 2], crafted[k + 3]);
        } else {
#pragma unroll
          for (int k = 0; k < VEC; ++k)
            if (c0 + k < d) dst[k] = crafted[k];
        }
      } else {
        if (v16) {
          uint32_t w[VEC / 2 > 0 ? VEC / 2 : 1];
#pragma unroll
          for (int k = 0; k + 1 < VEC; k += 2) w[k / 2] = bits16(from_f32<W>(crafted[k])) | (bits16(from_f32<W>(crafted[k + 1])) << 16);
#pragma unroll
          for (int k = 0; k + 8 <= VEC; k += 8)
            *reinterpret_cast<uint4*>(dst + k) = make_uint4(w[k / 2], w[k / 2 + 1], w[k / 2 + 2], w[k / 2 + 3]);
        } else {
#pragma unroll
          for (int k = 0; k < VEC; ++k)
            if (c0 + k < d) dst[k] = from_f32<W>(crafted[k]);
        }
      }
    }
  }
}

template <typename T, int VEC, bool COHERENT>
__global__ void __launch_bounds__(kBlock)
alie_kernel(const T* G, int f, int64_t d, int64_t ld, float z, float* __restrict__ mu_out,
            float* __restrict__ sigma_out, float* __restrict__ crafted_out, float* bcast, int64_t bcast_ld,
            int64_t g_batch, int64_t out_batch, int64_t bcast_batch, const ProblemParams* __restrict__ each) {
  alie_body<T, VEC, COHERENT, float>(G, f, d, ld, z, mu_out, sigma_out, crafted_out, bcast, bcast_ld, g_batch, out_batch,
                                     bcast_batch, each);
}

// ALIE of a 16-bit matrix whose crafted vector is written back into that matrix (afl_alie_batched_dev): the same
// statistics as alie_kernel, and the rows written in T.
template <typename T, int VEC, bool COHERENT>
__global__ void __launch_bounds__(kBlock)
alie_write16_kernel(const T* G, int f, int64_t d, int64_t ld, float z, float* __restrict__ mu_out,
                    float* __restrict__ sigma_out, float* __restrict__ crafted_out, T* bcast, int64_t bcast_ld,
                    int64_t g_batch, int64_t out_batch, int64_t bcast_batch, const ProblemParams* __restrict__ each) {
  alie_body<T, VEC, COHERENT, T>(G, f, d, ld, z, mu_out, sigma_out, crafted_out, bcast, bcast_ld, g_batch, out_batch,
                                 bcast_batch, each);
}

template <typename T>
__global__ void __launch_bounds__(kBlock)
gather_row_kernel(const T* __restrict__ G, int n, int64_t d, int64_t ld, const int* __restrict__ idx_dev,
                  float* __restrict__ out) {
  int idx = *idx_dev;
  if (idx < 0) idx += n;            // the reference's users_grads[-1] when nobody wins
  if (idx < 0 || idx >= n) return;
  const T* row = G + static_cast<int64_t>(idx) * ld;
  for (int64_t c = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x; c < d;
       c += static_cast<int64_t>(gridDim.x) * kBlock)
    out[c] = load_pack<T, 1>(row + c).v[0];
}

__global__ void __launch_bounds__(kBlock)
momentum_kernel(float* __restrict__ w, float* __restrict__ v, const float* __restrict__ g, int64_t d, float momentum,
                float lr, const float* __restrict__ lr_each) {
  // lr_each: row blockIdx.y of [batch, d] rows at its own learning rate (the scalar call's grid has one row)
  if (lr_each) {
    const int64_t off = static_cast<int64_t>(blockIdx.y) * d;
    w += off; v += off; g += off;
    lr = lr_each[blockIdx.y];
  }
  for (int64_t c = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x; c < d;
       c += static_cast<int64_t>(gridDim.x) * kBlock) {
    // server.py:89  velocity = momentum*velocity - lr*grads  (two products, one subtraction, fp32)
    const float nv = __fsub_rn(__fmul_rn(momentum, v[c]), __fmul_rn(lr, g[c]));
    v[c] = nv;
    w[c] = __fadd_rn(w[c], nv);                      // server.py:90
  }
}

// np.clip(v, lo, hi) = minimum(maximum(v, lo), hi) with NumPy's NaN propagation (backdoor.py:62-63).
__device__ __forceinline__ float np_clip(float v, float lo, float hi) {
  float r = fminf(fmaxf(v, lo), hi);
  if (v != v || lo != lo || hi != hi) r = __int_as_float(0x7fc00000);
  return r;
}

// ALIE band: lo = mu - z*sigma, hi = mu + z*sigma (fp32 product, fp32 sum: the roundings of
// `grads_mean -/+ num_std * grads_stdev`).  x == nullptr: out = lo (malicious.py:35, DriftAttack);
// otherwise out = np_clip(x, lo, hi) (backdoor.py:62-63).  out may alias mu or x (each element is read before it is
// written).
__global__ void __launch_bounds__(kBlock)
band_kernel(const float* mu, const float* sigma, float z, const float* x, float* out, int64_t d) {
  for (int64_t c = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x; c < d;
       c += static_cast<int64_t>(gridDim.x) * kBlock) {
    const float m = mu[c], zs = __fmul_rn(z, sigma[c]);
    const float lo = __fsub_rn(m, zs);
    if (x == nullptr) { out[c] = lo; continue; }
    const float hi = __fadd_rn(m, zs);
    out[c] = np_clip(x[c], lo, hi);
  }
}

// ---- backdoor crafting (backdoor.py:52-63) of a batch, problem b = blockIdx.y with lr = (float)learning_rate, z and f
// from its table row; [batch][d] fp32 vectors at b * d.  The caller's model training (backdoor.py:56) runs between
// the two kernels, so the crafting is two element-wise passes around it.
//
// start: initial = w - mu * lr (backdoor.py:54), w at b * w_batch (0: one vector shared by every problem).
__global__ void __launch_bounds__(kBlock)
backdoor_start_kernel(const float* __restrict__ mu, const float* __restrict__ w, int64_t w_batch, int64_t d,
                      const ProblemParams* __restrict__ each, float* __restrict__ initial) {
  const int64_t o = static_cast<int64_t>(blockIdx.y) * d;
  const float lr = each[blockIdx.y].lr;
  w += blockIdx.y * w_batch;
  for (int64_t c = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x; c < d;
       c += static_cast<int64_t>(gridDim.x) * kBlock)
    initial[o + c] = __fsub_rn(w[c], __fmul_rn(mu[o + c], lr));
}

// finish, for a problem that writes (f > 0, z != 0), with mal = the trained parameters (mal + b * mal_batch):
//   step = mu * lr; new_params = mal + step (backdoor.py:59); new_grads = (initial - new_params) / lr (backdoor.py:60,
//   IEEE division); crafted = np_clip(new_grads, mu - z*sigma, mu + z*sigma) (backdoor.py:62-63, band_kernel's roundings)
// and, with bcast, crafted over rows 0..f-1 of bcast + b * bcast_batch (server.py:82-83).  Any other problem reads no
// mal and writes no row: crafted = mu (z = 0: the statistics only; f = 0: mu is NaN).
__global__ void __launch_bounds__(kBlock)
backdoor_finish_kernel(const float* __restrict__ mu, const float* __restrict__ sigma, const float* __restrict__ initial,
                       const float* mal, int64_t mal_batch, int64_t d, const ProblemParams* __restrict__ each,
                       float* __restrict__ crafted_out, float* bcast, int64_t bcast_batch, int64_t bcast_ld) {
  const ProblemParams& q = each[blockIdx.y];
  const int64_t o = static_cast<int64_t>(blockIdx.y) * d;
  const bool write = q.write != 0;
  const int f = q.f;
  const float lr = q.lr, z = q.z;
  mal += blockIdx.y * mal_batch;
  if (bcast) bcast += blockIdx.y * bcast_batch;
  for (int64_t c = static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x; c < d;
       c += static_cast<int64_t>(gridDim.x) * kBlock) {
    const float m = mu[o + c];
    float r = m;
    if (write) {
      const float step = __fmul_rn(m, lr);
      const float g = __fdiv_rn(__fsub_rn(initial[o + c], __fadd_rn(mal[c], step)), lr);
      const float zs = __fmul_rn(z, sigma[o + c]);
      r = np_clip(g, __fsub_rn(m, zs), __fadd_rn(m, zs));
      if (bcast)
        for (int rr = 0; rr < f; ++rr) bcast[static_cast<int64_t>(rr) * bcast_ld + c] = r;
    }
    crafted_out[o + c] = r;
  }
}

// ---- attack-success metrics (metrics.py, SURVEY 8d "Attack-success (C5)"): how far an aggregate is from the mean of
// the honest clients, ||a - h|| / ||h||, and whether a selection holds malicious clients.  The malicious clients are
// rows 0..f-1 (main.py:28), so the honest ones are rows f..n-1, a different range per problem of a per-problem batch.
//
// A thread owns V adjacent columns (4 for fp32, 8 for the 16-bit formats) whatever the pitch: with an aligned base
// and pitch (VL) it takes them with one 16-byte load per row, otherwise with V scalar loads.  A tile is the kBlock * V
// columns of one CTA, so the tile count, and with it the order of every sum below, depends on d and the dtype only.
template <typename T, int V, bool VL>
__device__ __forceinline__ Pack<V> load_cols(const T* p, int64_t c0, int64_t d) {
  if constexpr (VL) {
    return load_pack<T, V>(p);
  } else {
    Pack<V> r;
#pragma unroll
    for (int k = 0; k < V; ++k) r.v[k] = c0 + k < d ? load_pack<T, 1>(p + k).v[0] : 0.f;
    return r;
  }
}

// Sums of a and b over the CTA in thread 0: lanes by butterfly, then the warps in warp order.  No atomics: the
// order is fixed.
__device__ __forceinline__ void cta_sum2(double& a, double& b) {
  __shared__ double s[2][kBlock / 32];
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane_id() == 0) { s[0][threadIdx.x / 32] = a; s[1][threadIdx.x / 32] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = s[0][0]; b = s[1][0];
#pragma unroll
    for (int w = 1; w < kBlock / 32; ++w) { a += s[0][w]; b += s[1][w]; }
  }
}

// cta_sum2 with a third sum: each of the three takes cta_sum2's order, so a and b come out as cta_sum2 gives them.
__device__ __forceinline__ void cta_sum3(double& a, double& b, double& c) {
  __shared__ double s[3][kBlock / 32];
  a = warp_sum(a);
  b = warp_sum(b);
  c = warp_sum(c);
  if (lane_id() == 0) { s[0][threadIdx.x / 32] = a; s[1][threadIdx.x / 32] = b; s[2][threadIdx.x / 32] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = s[0][0]; b = s[1][0]; c = s[2][0];
#pragma unroll
    for (int w = 1; w < kBlock / 32; ++w) { a += s[0][w]; b += s[1][w]; c += s[2][w]; }
  }
}

// h = mean of rows f..n-1: mean_kernel's sequential fp32 row sum and one IEEE division on that row range, so h is
// afl_mean of G[f:] bit for bit.  a = the aggregate: agg[b] (fp32, pitch d), or row idx[b] of G[b] upcast to fp32
// (Krum's result, read in place).  partial[b][tile] = (sum (a - h)^2, sum h^2) over the tile's columns in float64; the
// differences and squares are formed from the fp32 values as float64, so nothing cancels.  f >= n (no honest row)
// reads no row and gives h = 0 / 0 = NaN; an idx outside [0, n) reads no row and gives a = NaN.  partial == NULL:
// only honest_out is wanted.  kRows (a ragged batch): problem b has each[b].tm.n_rows rows instead of n.
// kTrace (afl_attack_trace_dev, agg given): also sum (r0 - h)^2 with r0 = row 0 when f > 0 (0 otherwise), formed as
// (a - h)^2 is, so that sum equals the first with a = row 0; partial is then read as double[3] per (problem, tile).
template <typename T, int V, bool VL, bool kRows, bool kTrace = false>
__global__ void __launch_bounds__(kBlock)
honest_deviation_kernel(const T* __restrict__ G, int n, int64_t d, int64_t ld, int64_t g_batch, int f,
                        const ProblemParams* __restrict__ each, const float* __restrict__ agg,
                        const int* __restrict__ idx, float* __restrict__ honest_out, double2* __restrict__ partial) {
  constexpr int U = VL ? kUnroll : 2;                 // V scalar loads per row: fewer rows in flight
  const int b = blockIdx.y;
  if (each) f = each[b].f;
  if constexpr (kRows) n = each[b].tm.n_rows;
  f = f < n ? f : n;
  const int64_t c0 = (static_cast<int64_t>(blockIdx.x) * kBlock + threadIdx.x) * V;
  double sd = 0.0, sh = 0.0;
  [[maybe_unused]] double sm = 0.0;
  if (c0 < d) {
    const T* p = G + b * g_batch + c0;
    float acc[V];
#pragma unroll
    for (int k = 0; k < V; ++k) acc[k] = 0.f;
    int r = f;
    for (; r + U <= n; r += U) {
      Pack<V> t[U];
#pragma unroll
      for (int u = 0; u < U; ++u) t[u] = load_cols<T, V, VL>(p + static_cast<int64_t>(r + u) * ld, c0, d);
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int k = 0; k < V; ++k) acc[k] = __fadd_rn(acc[k], t[u].v[k]);
    }
    for (; r < n; ++r) {
      Pack<V> t = load_cols<T, V, VL>(p + static_cast<int64_t>(r) * ld, c0, d);
#pragma unroll
      for (int k = 0; k < V; ++k) acc[k] = __fadd_rn(acc[k], t.v[k]);
    }
    Pack<V> a;
#pragma unroll
    for (int k = 0; k < V; ++k) a.v[k] = __int_as_float(0x7fc00000);
    if (idx) {
      const int i = idx[b];
      if (i >= 0 && i < n) a = load_cols<T, V, VL>(p + static_cast<int64_t>(i) * ld, c0, d);
    } else if (agg) {
#pragma unroll
      for (int k = 0; k < V; ++k)
        if (c0 + k < d) a.v[k] = __ldg(agg + b * d + c0 + k);
    }
    [[maybe_unused]] Pack<V> m;
    if constexpr (kTrace) {
      if (f > 0) m = load_cols<T, V, VL>(p, c0, d);
    }
    const float fn = static_cast<float>(n - f);
    const int64_t o = b * d + c0;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      if (c0 + k < d) {
        const float h = __fdiv_rn(acc[k], fn);
        if (honest_out) honest_out[o + k] = h;
        const double hd = static_cast<double>(h), df = static_cast<double>(a.v[k]) - hd;
        sd = fma(df, df, sd);
        sh = fma(hd, hd, sh);
        if constexpr (kTrace) {
          if (f > 0) { const double dm = static_cast<double>(m.v[k]) - hd; sm = fma(dm, dm, sm); }
        }
      }
    }
  }
  if constexpr (kTrace) {
    cta_sum3(sd, sh, sm);
    if (threadIdx.x == 0) {
      double* q = reinterpret_cast<double*>(partial) + 3 * (static_cast<int64_t>(b) * gridDim.x + blockIdx.x);
      q[0] = sd; q[1] = sh; q[2] = sm;
    }
  } else {
    if (!partial) return;
    cta_sum2(sd, sh);
    if (threadIdx.x == 0) partial[static_cast<int64_t>(b) * gridDim.x + blockIdx.x] = make_double2(sd, sh);
  }
}

// One CTA per problem: thread t adds tiles t, t + kBlock, ... in that order, then cta_sum2.  The order depends on
// the tile count only.  dev_out[b] = (float)sqrt(sum (a - h)^2 / sum h^2); sums_out[b] = the two float64 sums, which
// add across column shards.
__global__ void __launch_bounds__(kBlock)
deviation_finish_kernel(const double2* __restrict__ partial, int tiles, float* __restrict__ dev_out,
                        double* __restrict__ sums_out) {
  const int b = blockIdx.x;
  const double2* p = partial + static_cast<int64_t>(b) * tiles;
  double sd = 0.0, sh = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kBlock) { sd += p[t].x; sh += p[t].y; }
  cta_sum2(sd, sh);
  if (threadIdx.x == 0) {
    if (sums_out) { sums_out[2 * b] = sd; sums_out[2 * b + 1] = sh; }
    if (dev_out) dev_out[b] = static_cast<float>(sqrt(sd / sh));
  }
}

// One thread per problem.  krum_hit[b] = 0 <= idx[b] < f_b (metrics.krum_attack_success).  Over row b of sel
// (sel_ld entries; -1 = failed round, -2 = no such round): sel_count[b] = entries >= 0, mal_count[b] = entries in
// [0, f_b) (metrics.bulyan_attack_success is mal_count / max(1, sel_count)).
__global__ void __launch_bounds__(kBlock)
selection_stats_kernel(int batch, int f, const ProblemParams* __restrict__ each, const int* __restrict__ idx,
                       const int* __restrict__ sel, int sel_ld, int* __restrict__ krum_hit, int* __restrict__ mal_count,
                       int* __restrict__ sel_count) {
  const int b = blockIdx.x * kBlock + threadIdx.x;
  if (b >= batch) return;
  if (each) f = each[b].f;
  if (krum_hit) { const int i = idx[b]; krum_hit[b] = i >= 0 && i < f; }
  if (sel) {
    int mal = 0, cnt = 0;
    for (int j = 0; j < sel_ld; ++j) {
      const int i = sel[static_cast<int64_t>(b) * sel_ld + j];
      cnt += i >= 0;
      mal += i >= 0 && i < f;
    }
    if (mal_count) mal_count[b] = mal;
    if (sel_count) sel_count[b] = cnt;
  }
}

// afl_attack_trace_dev's finish, one CTA per problem: deviation_finish_kernel's order on three sums, then entry
// [*slot][b] of each given table (pitch table_ld): agg_dev = sqrt(sum (a - h)^2 / sum h^2), mal_dev the same with row 0
// (NaN when f_b = 0), idx_out = idx[b], and selection_stats_kernel's two counts.  A slot outside [0, n_slots) writes
// nothing.
__global__ void __launch_bounds__(kBlock)
trace_finish_kernel(const double* __restrict__ partial, int tiles, const ProblemParams* __restrict__ each,
                    const int* __restrict__ slot, int n_slots, int64_t table_ld, const int* __restrict__ idx,
                    const int* __restrict__ sel, int sel_ld, float* __restrict__ agg_dev, float* __restrict__ mal_dev,
                    int* __restrict__ idx_out, int* __restrict__ mal_count, int* __restrict__ sel_count) {
  const int b = blockIdx.x;
  const int s = *slot;
  if (s < 0 || s >= n_slots) return;                   // the whole CTA, before any barrier
  const double* p = partial + 3 * static_cast<int64_t>(b) * tiles;
  double sd = 0.0, sh = 0.0, sm = 0.0;
  for (int t = threadIdx.x; t < tiles; t += kBlock) { sd += p[3 * t]; sh += p[3 * t + 1]; sm += p[3 * t + 2]; }
  cta_sum3(sd, sh, sm);
  if (threadIdx.x != 0) return;
  const int f = each[b].f;
  const int64_t o = static_cast<int64_t>(s) * table_ld + b;
  if (agg_dev) agg_dev[o] = static_cast<float>(sqrt(sd / sh));
  if (mal_dev) mal_dev[o] = f > 0 ? static_cast<float>(sqrt(sm / sh)) : __int_as_float(0x7fc00000);
  if (idx_out) idx_out[o] = idx[b];
  if (sel) {
    int mal = 0, cnt = 0;
    for (int j = 0; j < sel_ld; ++j) {
      const int i = sel[static_cast<int64_t>(b) * sel_ld + j];
      cnt += i >= 0;
      mal += i >= 0 && i < f;
    }
    if (mal_count) mal_count[o] = mal;
    if (sel_count) sel_count[o] = cnt;
  }
}

// 16-byte loads need an aligned base, pitch and (batch > 1) batch pitch
static bool vec_ok(const void* G, int64_t ld, int dtype, int batch, int64_t g_batch) {
  const int64_t es = dtype == AFL_F32 ? 4 : 2;
  return (reinterpret_cast<uintptr_t>(G) % 16 == 0) && ((ld * es) % 16 == 0) && (batch == 1 || (g_batch * es) % 16 == 0);
}

// rows (device, may be NULL): a ragged batch, problem b averaging rows 0..rows[b].tm.n_rows-1 (at most n).
int mean_batched(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, int batch, int64_t g_batch,
                 int64_t out_batch, cudaStream_t stream, const ProblemParams* rows) {
  if (!G || !out || n < 1 || d < 1 || ld < d) { set_error("afl_mean: bad argument"); return AFL_ERR_BAD_ARG; }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_mean: dtype"); return AFL_ERR_UNSUPPORTED; }
  const bool v = vec_ok(G, ld, dtype, batch, g_batch);
  const int vec = v ? (dtype == AFL_F32 ? 4 : 8) : 1;
  const dim3 grid(static_cast<unsigned>(ceil_div64(ceil_div64(d, vec), kBlock)), batch);
  ProfScope ps("mean", stream);
#define AFL_MEAN_LAUNCH(T, V)                                                                                            \
  do {                                                                                                                   \
    if (rows) mean_kernel<T, V, true><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), n, d, ld, out, g_batch, out_batch, rows); \
    else mean_kernel<T, V, false><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), n, d, ld, out, g_batch, out_batch, nullptr); \
  } while (0)
  if (dtype == AFL_F32) {
    if (v) AFL_MEAN_LAUNCH(float, 4);
    else AFL_MEAN_LAUNCH(float, 1);
  } else if (dtype == AFL_BF16) {
    if (v) AFL_MEAN_LAUNCH(__nv_bfloat16, 8);
    else AFL_MEAN_LAUNCH(__nv_bfloat16, 1);
  } else {
    if (v) AFL_MEAN_LAUNCH(__half, 8);
    else AFL_MEAN_LAUNCH(__half, 1);
  }
#undef AFL_MEAN_LAUNCH
  AFL_LAUNCH_CHECK("mean_kernel");
  return AFL_OK;
}

int mean(const void* G, int n, int64_t d, int64_t ld, int dtype, float* out, cudaStream_t stream) {
  return mean_batched(G, n, d, ld, dtype, out, 1, 0, 0, stream, nullptr);
}

// `batch` problems: G + b * g_batch; mu/sigma/crafted + b * out_batch; bcast + b * bcast_batch.  each (device, may be
// NULL): per-problem f, z and write flag, f then being the largest problem's (0 allowed).
int alie_batched(const void* G, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
                 float* crafted_out, float* bcast, int64_t bcast_ld, int batch, int64_t g_batch, int64_t out_batch,
                 int64_t bcast_batch, cudaStream_t stream, const ProblemParams* each) {
  if (!G || f < (each ? 0 : 1) || d < 1 || ld < d || (bcast && bcast_ld < d)) { set_error("afl_alie: bad argument"); return AFL_ERR_BAD_ARG; }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_alie: dtype"); return AFL_ERR_UNSUPPORTED; }
  const bool v = vec_ok(G, ld, dtype, batch, g_batch);
  const int vec = v ? (dtype == AFL_F32 ? 4 : 8) : 1;
  const dim3 grid(static_cast<unsigned>(ceil_div64(ceil_div64(d, vec), kBlock)), batch);
  const float zf = static_cast<float>(z);
  ProfScope ps("alie", stream);
  // the reference writes the crafted vector back over the malicious rows (main.py:68 -> server.py:82-83): when the
  // broadcast target overlaps the input (any problem's), read it coherently (no ld.global.nc on memory this launch writes)
  const int64_t last = static_cast<int64_t>(batch - 1);
  const uintptr_t g0 = reinterpret_cast<uintptr_t>(G), g1 = g0 + static_cast<uintptr_t>((last * g_batch + static_cast<int64_t>(f - 1) * ld + d) * (dtype == AFL_F32 ? 4 : 2));
  const uintptr_t b0 = reinterpret_cast<uintptr_t>(bcast), b1 = b0 + static_cast<uintptr_t>((last * bcast_batch + static_cast<int64_t>(f - 1) * bcast_ld + d) * 4);
  const bool coh = bcast && f > 0 && b0 < g1 && g0 < b1;
#define AFL_ALIE_LAUNCH(T, V, C) alie_kernel<T, V, C><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), f, d, ld, zf, mu_out, sigma_out, crafted_out, bcast, bcast_ld, g_batch, out_batch, bcast_batch, each)
  if (dtype == AFL_F32) {
    if (v) { if (coh) AFL_ALIE_LAUNCH(float, 4, true); else AFL_ALIE_LAUNCH(float, 4, false); }
    else { if (coh) AFL_ALIE_LAUNCH(float, 1, true); else AFL_ALIE_LAUNCH(float, 1, false); }
  } else if (dtype == AFL_BF16) {
    if (v) { if (coh) AFL_ALIE_LAUNCH(__nv_bfloat16, 8, true); else AFL_ALIE_LAUNCH(__nv_bfloat16, 8, false); }
    else { if (coh) AFL_ALIE_LAUNCH(__nv_bfloat16, 1, true); else AFL_ALIE_LAUNCH(__nv_bfloat16, 1, false); }
  } else {
    if (v) { if (coh) AFL_ALIE_LAUNCH(__half, 8, true); else AFL_ALIE_LAUNCH(__half, 8, false); }
    else { if (coh) AFL_ALIE_LAUNCH(__half, 1, true); else AFL_ALIE_LAUNCH(__half, 1, false); }
  }
#undef AFL_ALIE_LAUNCH
  AFL_LAUNCH_CHECK("alie_kernel");
  return AFL_OK;
}

// alie_batched with a table (each required) and bcast in G's dtype (afl_alie_batched_dev).  f_bound >= every f_b (the
// slot's row count): it only widens the overlap test that picks coherent loads, which changes no value.
int alie_batched_dev(const void* G, int f_bound, int64_t d, int64_t ld, int dtype, float* mu_out, float* sigma_out,
                     float* crafted_out, void* bcast, int64_t bcast_ld, int batch, int64_t g_batch, int64_t out_batch,
                     int64_t bcast_batch, cudaStream_t stream, const ProblemParams* each) {
  if (dtype == AFL_F32 || !bcast)
    return alie_batched(G, f_bound, d, ld, dtype, 0.0, mu_out, sigma_out, crafted_out, static_cast<float*>(bcast),
                        bcast_ld, batch, g_batch, out_batch, bcast_batch, stream, each);
  if (!G || !each || f_bound < 0 || d < 1 || ld < d || bcast_ld < d) { set_error("afl_alie: bad argument"); return AFL_ERR_BAD_ARG; }
  if (dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_alie: dtype"); return AFL_ERR_UNSUPPORTED; }
  const bool v = vec_ok(G, ld, dtype, batch, g_batch);
  const int vec = v ? 8 : 1;
  const dim3 grid(static_cast<unsigned>(ceil_div64(ceil_div64(d, vec), kBlock)), batch);
  ProfScope ps("alie", stream);
  const int64_t last = static_cast<int64_t>(batch - 1);
  const uintptr_t g0 = reinterpret_cast<uintptr_t>(G), g1 = g0 + static_cast<uintptr_t>((last * g_batch + static_cast<int64_t>(f_bound - 1) * ld + d) * 2);
  const uintptr_t b0 = reinterpret_cast<uintptr_t>(bcast), b1 = b0 + static_cast<uintptr_t>((last * bcast_batch + static_cast<int64_t>(f_bound - 1) * bcast_ld + d) * 2);
  const bool coh = f_bound > 0 && b0 < g1 && g0 < b1;
#define AFL_ALIE16_LAUNCH(T, V, C) alie_write16_kernel<T, V, C><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), f_bound, d, ld, 0.f, mu_out, sigma_out, crafted_out, static_cast<T*>(bcast), bcast_ld, g_batch, out_batch, bcast_batch, each)
  if (dtype == AFL_BF16) {
    if (v) { if (coh) AFL_ALIE16_LAUNCH(__nv_bfloat16, 8, true); else AFL_ALIE16_LAUNCH(__nv_bfloat16, 8, false); }
    else { if (coh) AFL_ALIE16_LAUNCH(__nv_bfloat16, 1, true); else AFL_ALIE16_LAUNCH(__nv_bfloat16, 1, false); }
  } else {
    if (v) { if (coh) AFL_ALIE16_LAUNCH(__half, 8, true); else AFL_ALIE16_LAUNCH(__half, 8, false); }
    else { if (coh) AFL_ALIE16_LAUNCH(__half, 1, true); else AFL_ALIE16_LAUNCH(__half, 1, false); }
  }
#undef AFL_ALIE16_LAUNCH
  AFL_LAUNCH_CHECK("alie_write16_kernel");
  return AFL_OK;
}

int alie(const void* G, int f, int64_t d, int64_t ld, int dtype, double z, float* mu_out, float* sigma_out,
         float* crafted_out, float* bcast, int64_t bcast_ld, cudaStream_t stream) {
  return alie_batched(G, f, d, ld, dtype, z, mu_out, sigma_out, crafted_out, bcast, bcast_ld, 1, 0, 0, 0, stream, nullptr);
}

int gather_row(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* idx_dev, float* out,
               cudaStream_t stream) {
  if (!G || !idx_dev || !out || n < 1 || d < 1 || ld < d) { set_error("afl_gather_row: bad argument"); return AFL_ERR_BAD_ARG; }
  int64_t blocks = ceil_div64(d, kBlock);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (dtype == AFL_F32)
    gather_row_kernel<float><<<static_cast<unsigned>(blocks), kBlock, 0, stream>>>(static_cast<const float*>(G), n, d, ld, idx_dev, out);
  else if (dtype == AFL_BF16)
    gather_row_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), kBlock, 0, stream>>>(static_cast<const __nv_bfloat16*>(G), n, d, ld, idx_dev, out);
  else if (dtype == AFL_F16)
    gather_row_kernel<__half><<<static_cast<unsigned>(blocks), kBlock, 0, stream>>>(static_cast<const __half*>(G), n, d, ld, idx_dev, out);
  else { set_error("afl_gather_row: dtype"); return AFL_ERR_UNSUPPORTED; }
  AFL_LAUNCH_CHECK("gather_row_kernel");
  return AFL_OK;
}

// Column tiles of honest_deviation_kernel: kBlock threads of 4 (fp32) or 8 (bf16, fp16) columns.
int64_t deviation_tiles(int64_t d, int dtype) { return ceil_div64(d, kBlock * (dtype == AFL_F32 ? 4 : 8)); }

// The three metric kernels on `batch` problems (arguments checked by the caller, capi.cu).  The deviation pass runs
// when dev_out, sums_out or honest_out is wanted, the finish for the first two, the selection statistics when
// krum_hit or sel is given.  partial: double2[batch][deviation_tiles].  rows (each required): a ragged batch, problem b
// having each[b].tm.n_rows rows.
int attack_metrics(const void* G, int batch, int64_t g_batch, int n, int64_t d, int64_t ld, int dtype, int f,
                   const ProblemParams* each, const float* agg, const int* idx, const int* sel, int sel_ld,
                   float* dev_out, double* sums_out, float* honest_out, int* krum_hit, int* mal_count, int* sel_count,
                   void* partial, cudaStream_t stream, bool rows) {
  const bool sums = dev_out || sums_out;
  if (sums || honest_out) {
    const int tiles = static_cast<int>(deviation_tiles(d, dtype));
    const dim3 grid(tiles, batch);
    const bool v = vec_ok(G, ld, dtype, batch, g_batch);
    double2* part = sums ? static_cast<double2*>(partial) : nullptr;
    {
      ProfScope ps("honest_deviation", stream);
#define AFL_DEV_LAUNCH(T, V, VL)                                                                                          \
  do {                                                                                                                   \
    if (rows) honest_deviation_kernel<T, V, VL, true><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), n, d, ld, g_batch, f, each, agg, idx, honest_out, part); \
    else honest_deviation_kernel<T, V, VL, false><<<grid, kBlock, 0, stream>>>(static_cast<const T*>(G), n, d, ld, g_batch, f, each, agg, idx, honest_out, part); \
  } while (0)
      if (dtype == AFL_F32) {
        if (v) AFL_DEV_LAUNCH(float, 4, true);
        else AFL_DEV_LAUNCH(float, 4, false);
      } else if (dtype == AFL_BF16) {
        if (v) AFL_DEV_LAUNCH(__nv_bfloat16, 8, true);
        else AFL_DEV_LAUNCH(__nv_bfloat16, 8, false);
      } else {
        if (v) AFL_DEV_LAUNCH(__half, 8, true);
        else AFL_DEV_LAUNCH(__half, 8, false);
      }
#undef AFL_DEV_LAUNCH
      AFL_LAUNCH_CHECK("honest_deviation_kernel");
    }
    if (sums) {
      deviation_finish_kernel<<<batch, kBlock, 0, stream>>>(part, tiles, dev_out, sums_out);
      AFL_LAUNCH_CHECK("deviation_finish_kernel");
    }
  }
  if (krum_hit || sel) {
    selection_stats_kernel<<<static_cast<unsigned>(ceil_div64(batch, kBlock)), kBlock, 0, stream>>>(
        batch, f, each, idx, sel, sel_ld, krum_hit, mal_count, sel_count);
    AFL_LAUNCH_CHECK("selection_stats_kernel");
  }
  return AFL_OK;
}

// afl_attack_trace_dev's two kernels on `batch` fp32 problems (arguments checked by the caller, capi.cu): the trace
// instance of honest_deviation_kernel against agg, then trace_finish_kernel.  partial: double[batch][tiles][3].
int attack_trace(const float* G, int batch, int64_t g_batch, int n, int64_t d, int64_t ld, const ProblemParams* each,
                 const float* agg, const int* idx, const int* sel, int sel_ld, const int* slot, int n_slots,
                 int64_t table_ld, float* agg_dev, float* mal_dev, int* idx_out, int* mal_count, int* sel_count,
                 void* partial, cudaStream_t stream, bool rows) {
  const int tiles = static_cast<int>(deviation_tiles(d, AFL_F32));
  const dim3 grid(tiles, batch);
  const bool v = vec_ok(G, ld, AFL_F32, batch, g_batch);
  double2* part = static_cast<double2*>(partial);
  ProfScope ps("attack_trace", stream);
#define AFL_TRACE_LAUNCH(VL)                                                                                             \
  do {                                                                                                                   \
    if (rows) honest_deviation_kernel<float, 4, VL, true, true><<<grid, kBlock, 0, stream>>>(G, n, d, ld, g_batch, 0, each, agg, nullptr, nullptr, part); \
    else honest_deviation_kernel<float, 4, VL, false, true><<<grid, kBlock, 0, stream>>>(G, n, d, ld, g_batch, 0, each, agg, nullptr, nullptr, part); \
  } while (0)
  if (v) AFL_TRACE_LAUNCH(true);
  else AFL_TRACE_LAUNCH(false);
#undef AFL_TRACE_LAUNCH
  AFL_LAUNCH_CHECK("honest_deviation_kernel");
  trace_finish_kernel<<<batch, kBlock, 0, stream>>>(static_cast<const double*>(partial), tiles, each, slot, n_slots,
                                                     table_ld, idx, sel, sel_ld, agg_dev, mal_dev, idx_out, mal_count,
                                                     sel_count);
  AFL_LAUNCH_CHECK("trace_finish_kernel");
  return AFL_OK;
}

int momentum_step(float* w, float* v, const float* g, int64_t d, float momentum, float lr, cudaStream_t stream) {
  if (!w || !v || !g || d < 1) { set_error("afl_momentum_step: bad argument"); return AFL_ERR_BAD_ARG; }
  int64_t blocks = ceil_div64(d, kBlock);
  if (blocks > 132 * 16) blocks = 132 * 16;
  momentum_kernel<<<static_cast<unsigned>(blocks), kBlock, 0, stream>>>(w, v, g, d, momentum, lr, nullptr);
  AFL_LAUNCH_CHECK("momentum_kernel");
  return AFL_OK;
}

int momentum_step_batched(float* w, float* v, const float* g, int batch, int64_t d, float momentum, const float* lr,
                          cudaStream_t stream) {
  if (!w || !v || !g || !lr || batch < 1 || d < 1) {
    set_error("afl_momentum_step_batched: bad argument");
    return AFL_ERR_BAD_ARG;
  }
  if (batch > 65535) {
    set_error("afl_momentum_step_batched: batch <= 65535 rows (got %d)", batch);
    return AFL_ERR_UNSUPPORTED;
  }
  int64_t blocks = ceil_div64(d, kBlock);
  if (blocks > 132 * 16) blocks = 132 * 16;
  momentum_kernel<<<dim3(static_cast<unsigned>(blocks), batch), kBlock, 0, stream>>>(w, v, g, d, momentum, 0.f, lr);
  AFL_LAUNCH_CHECK("momentum_kernel");
  return AFL_OK;
}

int alie_band(const float* mu, const float* sigma, double z, const float* x, float* out, int64_t d,
              cudaStream_t stream) {
  if (!mu || !sigma || !out || d < 1) { set_error("afl_alie_band: bad argument"); return AFL_ERR_BAD_ARG; }
  int64_t blocks = ceil_div64(d, kBlock);
  if (blocks > 132 * 16) blocks = 132 * 16;
  band_kernel<<<static_cast<unsigned>(blocks), kBlock, 0, stream>>>(mu, sigma, static_cast<float>(z), x, out, d);
  AFL_LAUNCH_CHECK("band_kernel");
  return AFL_OK;
}

// Grid of the backdoor's element-wise passes: column blocks (capped, the kernels stride) x problems.
static dim3 backdoor_grid(int64_t d, int batch) {
  int64_t blocks = ceil_div64(d, kBlock);
  if (blocks > 132 * 16) blocks = 132 * 16;
  return dim3(static_cast<unsigned>(blocks), batch);
}

// The backdoor's statistics (afl_alie's per-problem pass on rows 0..f_b-1, nothing crafted or written), then initial.
// fmax: the largest f_b.  Arguments checked by the caller (capi.cu).
int backdoor_start(const void* G, int fmax, int64_t d, int64_t ld, int dtype, int batch, int64_t g_batch,
                   const ProblemParams* each, const float* w, int64_t w_batch, float* mu_out, float* sigma_out,
                   float* initial_out, cudaStream_t stream) {
  int rc = alie_batched(G, fmax, d, ld, dtype, 0.0, mu_out, sigma_out, nullptr, nullptr, 0, batch, g_batch, d, 0,
                        stream, each);
  if (rc) return rc;
  ProfScope ps("backdoor_start", stream);
  backdoor_start_kernel<<<backdoor_grid(d, batch), kBlock, 0, stream>>>(mu_out, w, w_batch, d, each, initial_out);
  AFL_LAUNCH_CHECK("backdoor_start_kernel");
  return AFL_OK;
}

int backdoor_finish(int batch, int64_t d, const ProblemParams* each, const float* mu, const float* sigma,
                    const float* initial, const float* mal, int64_t mal_batch, float* crafted_out, float* bcast,
                    int64_t bcast_batch, int64_t bcast_ld, cudaStream_t stream) {
  ProfScope ps("backdoor_finish", stream);
  backdoor_finish_kernel<<<backdoor_grid(d, batch), kBlock, 0, stream>>>(mu, sigma, initial, mal, mal_batch, d, each,
                                                                          crafted_out, bcast, bcast_batch, bcast_ld);
  AFL_LAUNCH_CHECK("backdoor_finish_kernel");
  return AFL_OK;
}

}  // namespace colstats
}  // namespace afl
