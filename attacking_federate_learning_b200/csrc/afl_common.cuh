// Shared device/host helpers for the sm_90a kernels: error plumbing, PTX wrappers for mbarrier,
// TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma) and small warp utilities.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/afl_b200.h"

#ifndef AFL_BAR_TIMEOUT_LOG2
#define AFL_BAR_TIMEOUT_LOG2 32
#endif

namespace afl {

// ------------------------------------------------------------------------------------------------
// host-side error plumbing
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
void count_launch(int n = 1);

#define AFL_CUDA(call)                                                        \
  do {                                                                        \
    cudaError_t _e = (call);                                                  \
    if (_e != cudaSuccess) return ::afl::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

#define AFL_LAUNCH_CHECK(name)                                                \
  do {                                                                        \
    ::afl::count_launch();                                                    \
    cudaError_t _e = cudaGetLastError();                                      \
    if (_e != cudaSuccess) return ::afl::cuda_fail(_e, name, __FILE__, __LINE__); \
  } while (0)

constexpr int kMaxDevices = 64;
int current_device();      // ordinal of the current device (0 when no device is visible)
int sm_count();            // SM count of the CURRENT device

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per device: remember it per (kernel, device).
template <typename K>
static inline cudaError_t ensure_dyn_smem(K kernel, int bytes, int (&done)[kMaxDevices]) {
  const int dev = current_device();
  if (done[dev] >= bytes) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done[dev] = bytes;
  return e;
}

constexpr int kMaxWorld = 16;            // ranks of one peer-exchange context (csrc/xgpu.cu)

// Trimmed-mean constants (csrc/trimmed_mean.cu, tmean::shape) of `n_rows` participating rows and a corrupted count.
struct TmShape {
  int n_rows;             // participating rows
  int keep;               // effective number of kept devs (python slice semantics applied), >= 0
  float med_density;      // 0.39894228 * n_rows (ranks per unit value at the centre of a unit Gaussian)
  float key_q;            // Gaussian guess of the |dev| threshold in sigmas
  float key_density;      // 2 * phi(key_q) * n_rows (ranks per unit |dev| at that threshold, unit sigma)
};

// One problem of a per-problem batched call (afl_defend_batched_each, afl_alie_batched_each): the values the single
// call derives on the host from that problem's corrupted_count and z.  The table of `batch` rows sits at the start of
// the caller's workspace; the kernels read row blockIdx.y (Bulyan's rounds: blockIdx.x) when handed a table.
struct ProblemParams {
  int f;                  // corrupted_count: Bulyan's first-round keep, ALIE's and the backdoor's rows
  int take;               // Krum: len(sorted(...)[:users_count - f])
  union {                 // a table serves either a defence or an attack, so the row keeps its 40 bytes
    int theta;            // Bulyan: users_count - 2f rounds
    float lr;             // backdoor: (float)learning_rate
  };
  int write;              // ALIE, backdoor: crafted is written over rows 0..f-1 (f > 0 and z != 0)
  float z;                // ALIE, backdoor: (float)z
  TmShape tm;             // TrimmedMean: n rows and f; Bulyan's second stage: theta rows and 2f
};

// Arguments of the Krum kernel (csrc/select.cu).  The row of distances comes from `dist` (a caller's fp32 table) when
// it is set, otherwise from the float64 d2 tables tab[0..world), summed in rank order; with world > 1 the kernel first
// waits until `flags` reach `epoch` and reads the peers' tables through their mappings.
struct KrumParams {
  const double* tab[kMaxWorld];
  const unsigned long long* flags;
  unsigned long long epoch;
  int world;
  const float* dist;
  int n, take;
  const ProblemParams* each;              // per-problem take, or NULL: `take` for every problem
  float* score;                           // [n]
  unsigned int* done;                     // last-CTA counter: zero at launch, reset by the kernel
  int* idx_dev;
  int* idx_host; int* status_host;        // mapped host words of the peer path, or NULL
};

// Optional CUDA-event bracket around a kernel launch (active only after afl_profile_enable(1)).
struct ProfScope {
  ProfScope(const char* name, cudaStream_t stream);
  ~ProfScope();
  const char* name_; cudaStream_t stream_; void* rec_;
};

// Operand formats of the tensor-core Gram kernel (csrc/gram_pair.cu)
enum GramMode { kModeBf16x2 = 0, kModeTf32x2 = 1, kModeBf16In = 2, kModeF16In = 3 };

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------
// small device utilities
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Streaming (read-once) global loads: bypass L1 allocation.
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ldg_stream_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t b16) { return __uint_as_float(b16 << 16); }
// fp16 in the low 16 bits -> fp32 (exact, subnormals and infinities included)
__device__ __forceinline__ float f16_bits_to_f32(uint32_t b16) {
  return __half2float(__ushort_as_half(static_cast<unsigned short>(b16)));
}

// ------------------------------------------------------------------------------------------------
// peer-memory exchange (csrc/xgpu.cu): epoch flags and the peers' tables
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ double ld_peer_f64(const double* p) {       // never served from a stale L1 line
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

// Wait (bounded) until every rank has published `epoch`.  Returns false on timeout.
__device__ __forceinline__ bool wait_flags(const unsigned long long* flags, int world, unsigned long long epoch) {
  __shared__ int s_ok;
  if (threadIdx.x == 0) s_ok = 1;
  __syncthreads();
  if (static_cast<int>(threadIdx.x) < world) {
    const long long t0 = clock64();
    while (ld_acquire_sys(flags + threadIdx.x) < epoch) {
      if (clock64() - t0 > (1ll << 33)) { s_ok = 0; break; }           // ~4 s: a peer died or never launched
    }
  }
  __syncthreads();
  return s_ok != 0;
}

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (launch error) instead of hanging the GPU.  No diagnostic printf: a function
// call anywhere in a kernel makes ptxas serialise its wgmma instructions.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > (1ll << AFL_BAR_TIMEOUT_LOG2)) __trap();   // ~2 s by default: no legitimate wait is that long
}

// Warp-level wait: one lane spins, the others sleep at the warp barrier and then observe the (already
// completed) phase with a single probe each, which gives every lane its own acquire.
__device__ __forceinline__ void mbar_wait_warp(uint64_t* bar, uint32_t parity) {
  if ((threadIdx.x & 31) == 0) mbar_wait(bar, parity);
  __syncwarp();
  mbar_wait(bar, parity);          // completes on the first probe; bounded like every other wait
}

// Explicit shared-space 16-byte accesses (a hand-aligned pointer into dynamic shared memory loses its
// address space and would otherwise compile to slow generic LD.E / ST.E).
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Fast-path wait: one probe by every lane (an already-completed phase costs a single try_wait); only if
// the phase is still pending does lane 0 spin while the others sleep at the warp barrier.
__device__ __forceinline__ void mbar_wait_fast(uint64_t* bar, uint32_t parity) {
  if (__all_sync(0xffffffffu, mbar_try_wait(bar, parity))) return;
  mbar_wait_warp(bar, parity);
}

// generic-proxy writes (st.shared) -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------------------------
// TMA
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 3-D tiled load, completes `bytes` on the mbarrier.  c0 = innermost (column) coord, c1 = row coord, c2 = problem.
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, uint64_t cache_policy) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "l"(cache_policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// ------------------------------------------------------------------------------------------------
// wgmma (Hopper warpgroup MMA): D[regs] (+)= A[smem desc] * B[smem desc]^T, fp32 accumulate, issued by all 128
// threads of a warpgroup
// ------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: K-major operand, 128-byte swizzle, rows of exactly 128 bytes, 8-row groups `sbo`
// bytes apart (the layout a TMA box of 128-byte rows writes with SWIZZLE_128B).  Fields: start>>4 [0,14) |
// LBO>>4 [16,30) (ignored for swizzled K-major) | SBO>>4 [32,46) | base offset 0 (1024-byte aligned atoms) |
// layout 1 = SWIZZLE_128B [62,64).  Advancing the start by 32 bytes steps along K inside the swizzled row.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr, uint32_t sbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across a wgmma_wait
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// m64n128: thread t of the warpgroup holds 64 accumulators; keep == 0 overwrites D instead of accumulating.
// AB = the operand type of both 16-bit operands: bf16 or f16 (fp16 clients, kModeF16In).
#define AFL_WGMMA_M64N128K16(NAME, AB)                                                                             \
  __device__ __forceinline__ void NAME(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t keep) {       \
    asm volatile(                                                                                                 \
        "{\n\t.reg .pred p;\n\t"                                                                                  \
        "setp.ne.b32 p, %66, 0;\n\t"                                                                              \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." AB "." AB " "                                              \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, " \
        "%64, %65, p, 1, 1, 0, 0;\n\t}\n"                                                                         \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),         \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),     \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),   \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),   \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),   \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),   \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),   \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])    \
        : "l"(a_desc), "l"(b_desc), "r"(keep));                                                                   \
  }
AFL_WGMMA_M64N128K16(wgmma_m64n128k16_bf16, "bf16")
AFL_WGMMA_M64N128K16(wgmma_m64n128k16_f16, "f16")
#undef AFL_WGMMA_M64N128K16
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t keep) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
      "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
      "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
      "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
      "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
      "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
      "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
      "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(keep));
}

// Centre of the bf16x2 Gram kernels: mean of the LAST `rows` clients (cref = first of those rows, pitch ld) over
// this lane's 4 consecutive columns starting at `col`.  Distances are translation invariant, so any centre is
// correct; a centre close to the clients' common component keeps ||g - c||^2 (which the dropped-term and
// accumulation biases scale with) of the order of the distances themselves.  Ids >= f are honest (main.py:28).
constexpr int kGramCenterRows = 8;
// A centre row with an inf in a column would turn every client's g - c there into inf or NaN: that column is not
// centred (c = 0), so only the rows that hold the inf get non-finite operands.
__device__ __forceinline__ float gram_center_finite(float c) { return isfinite(c) ? c : 0.f; }
__device__ __forceinline__ float4 gram_center_finite(float4 c) {
  return make_float4(gram_center_finite(c.x), gram_center_finite(c.y), gram_center_finite(c.z), gram_center_finite(c.w));
}
__device__ __forceinline__ float4 gram_center(const float* cref, int rows, int64_t ld, int64_t col, int64_t d) {
  // always kGramCenterRows loads, all issued before the first add (a runtime trip count would serialise 8 dependent
  // L2 round trips per k-block); with fewer clients the last row is simply counted more than once - any centre is valid
  float4 t[kGramCenterRows];
  if (col + 3 < d) {
#pragma unroll
    for (int r = 0; r < kGramCenterRows; ++r)
      t[r] = __ldg(reinterpret_cast<const float4*>(cref + static_cast<int64_t>(r < rows ? r : rows - 1) * ld + col));
  } else {
#pragma unroll
    for (int r = 0; r < kGramCenterRows; ++r) {
      const float* q = cref + static_cast<int64_t>(r < rows ? r : rows - 1) * ld + col;
      t[r] = make_float4(col < d ? __ldg(q) : 0.f, col + 1 < d ? __ldg(q + 1) : 0.f, col + 2 < d ? __ldg(q + 2) : 0.f, 0.f);
    }
  }
  float cx = 0.f, cy = 0.f, cz = 0.f, cw = 0.f;
#pragma unroll
  for (int r = 0; r < kGramCenterRows; ++r) { cx += t[r].x; cy += t[r].y; cz += t[r].z; cw += t[r].w; }
  const float inv = 1.0f / static_cast<float>(kGramCenterRows);
  return gram_center_finite(make_float4(cx * inv, cy * inv, cz * inv, cw * inv));
}


#endif  // __CUDACC__

}  // namespace afl
