// Coordinate-wise trimmed mean around the median (reference: defences.py:44-52) — also Bulyan's
// second stage (defences.py:70) through `row_index`.
//
// Per column:  med = median of the N values (even N: fl32 mean of the two middle ones);
//              dev = fl32(x - med); keep the k devs of smallest |dev|, ties in client (row) order;
//              out = fl32(fl32(sum(kept)/k) + med).
//
// Layout / mapping
//   * A CTA owns a tile of 64 bytes per row (16 fp32 or 32 bf16 / fp16 columns) x all rows.  Rows are read
//     with coalesced 16-byte loads (4 lanes per row segment) and scattered into shared memory in a
//     [word-column][slot-group][lane] order with an XOR on the slot-in-group index, so that both the
//     staging stores (STS.32) and the per-column reads (LDS.128) are bank-conflict free.
//   * One warp then owns one word-column: lane l holds rows l, l+32, l+64, ... in registers
//     (S slots per lane, S = 4, 8, 12, ..., 32: the smallest multiple of 4 with 32 S >= rows), so every pass over
//     the column is pure register arithmetic plus one warp reduction.  Rows past N are staged as +inf.
//   * Element formats (template parameter DT, an afl_dtype): fp32 occupies one word per column; bf16 and fp16 two
//     columns per word, unpacked to fp32 (exactly) as the column is loaded into registers, so everything after the
//     unpack is the fp32 arithmetic.
//   * Selection, fast path (select_fast): ONE fused pass per order statistic with a bracket [a, b) aimed from the
//     column's mean / sigma (median) or sigma and the normal quantile (|dev| threshold): it counts #{key < a}, sums
//     the devs below a, and marks the in-bracket slots in a per-lane bit mask (4-5 instructions per value, in PTX).
//     When the target rank is inside and <= 32 slots are marked, the candidates are re-read from the tile by slot
//     index, compacted to one per lane (shuffle scan) and sorted with a 15-stage shuffle bitonic network; otherwise
//     the bracket is re-aimed from the measured counts (about one column in four needs a second pass).
//   * Selection, general path (warp_select): interpolation search on counts with a min/max bisection fallback on the
//     integer image of the keys, which halves the bracket's image range per pass: at most 4 model passes + 32
//     bisection passes for any non-NaN column (heavy ties, non-Gaussian columns, values spread over every binade),
//     inside the loop's cap of 96; brackets of <= 32 elements are compacted by ballot
//     and ranked on (key, row), which makes the reference's stable tie rule exact.  In the fast path a tie group that
//     the keep boundary cuts (ALIE's f identical rows, bf16 value collisions) is resolved in row order with ballots on
//     the register-resident column (tie_sum).
//   * More than 1024 rows: trimmed_mean_large_kernel (shared-memory strip, bisection on the integer image of the keys).
//   * A batch (grid y) may carry a ProblemParams table: problem b then has its own participating rows, keep and pivot
//     constants (tm); rows past a problem's n_rows are staged as +inf like the rows past n_rows of a single call.  With
//     n <= 128 rows every problem runs trimmed_mean_kernel<4, DT, EACH> over grid y = problem.  Larger batches
//     (trimmed_mean_classes) run every problem in the instance that its own n_rows selects, as its single call does: one
//     launch per slot class present, grid y = the class's problems, problem P.perm[blockIdx.y] (CLASS).  The device-
//     parameter calls (trimmed_mean_classes_dev) read the class sizes from device memory instead: one persistent-grid
//     launch per class, every class, whose CTAs stride over the class's (problem, column tile) items (DEV).
#include <type_traits>

#include "afl_common.cuh"

namespace afl {
namespace tmean {

constexpr int kThreads = 256;
constexpr int kWarps = 8;
constexpr int kWordCols = 16;             // 32-bit words per staged row (64 bytes)
constexpr float kInf = __builtin_huge_valf();

struct Params {
  const void* G;
  const int* row_index;   // may be null
  float* out;
  int64_t d, ld;
  int n_total;            // rows of G (bounds for row_index)
  TmShape tm;             // participating rows, kept devs and the pivot model's constants
  const ProblemParams* each;    // per-problem tm (trimmed_mean_kernel<4, *> only), or NULL: `tm` for every problem
  int64_t g_batch, out_batch;   // problem blockIdx.y: G, out and row_index advance by these (elements)
  int ri_batch;
  int vec_ok;
};
// A class launch's arguments (trimmed_mean_kernel<S, DT, true, true>): Params and the class's problems (device).  A type
// of its own, so that Params and the kernels that take it keep their layout.
struct ClassParams : Params {
  const int* perm;
};
template <bool CLASS> using KernelParams = std::conditional_t<CLASS, ClassParams, Params>;

__device__ __forceinline__ int warp_sum_i(int v) { return __reduce_add_sync(0xffffffffu, v); }
__device__ __forceinline__ float warp_min_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Monotone map float -> uint32 (total order incl. negatives; NaN sorts last for positive payloads).
__device__ __forceinline__ uint32_t ord_bits(float x) {
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float from_ord_bits(uint32_t o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

// true row of register index ri (registers hold each 4-slot group permuted by jx, see staging)
__device__ __forceinline__ int row_of(int ri, int jx, int lane) { return (((ri & ~3) | ((ri & 3) ^ jx)) << 5) + lane; }

template <bool KEYS> __device__ __forceinline__ float keyof(float v) { return KEYS ? fabsf(v) : v; }

// One counting pass: c = #{key(v) < p} (warp total); for KEYS also s = this LANE's sum of v over those elements.
template <int S, bool KEYS>
__device__ __forceinline__ void count_pass(const float (&v)[S], float p, int& c, float& s) {
  int cc = 0;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    const bool b = keyof<KEYS>(v[i]) < p;
    cc += b ? 1 : 0;
    if (KEYS) ss += b ? v[i] : 0.f;
  }
  c = warp_sum_i(cc);
  if (KEYS) s = ss;                 // lane-local partial; reduced once at the very end
}

template <int S>
__device__ __forceinline__ float tie_sum(const float (&v)[S], float T, int need, int jx, int lane);

// Selection over a register-resident column (general path: any data, any bracket state).
//   KEYS = false : returns the order statistics of ranks r1 <= r2 (r2 <= r1 + 1) in a, b.
//   KEYS = true  : v holds devs, key = |dev|; r1 == r2 == keep-1; returns in `a` the sum of the `keep`
//                  devs of smallest key with ties resolved in row order.
template <int S, bool KEYS>
__device__ __forceinline__ void warp_select(const float (&v)[S], int n, int r1, int r2, float p0, float density,
                                            int lane, int jx, uint32_t* scratch, float lo, float hi, int c_lo, int c_hi,
                                            float sum_lo, float& a, float& b) {
  bool model = (density > 0.f) && (density < kInf) && (p0 == p0) && (fabsf(p0) < kInf) && (lo == -kInf) && (hi == kInf);
  float p = p0;
  a = b = __int_as_float(0x7fc00000);
  for (int iter = 0; iter < 96; ++iter) {
    const int inb = c_hi - c_lo;
    if (inb <= 32) {
      // ---- compact the bracket into this warp's smem scratch (ballot prefix), then rank every
      // candidate by counting (key, row) pairs below it: independent broadcast loads, no shuffles.
      unsigned long long* sk = reinterpret_cast<unsigned long long*>(scratch);      // [32] (ord(key) << 32) | row
      float* sp = reinterpret_cast<float*>(scratch + 64);                            // [32] payload
      sk[lane] = ~0ull;
      sp[lane] = 0.f;
      __syncwarp();
      int base = 0;
#pragma unroll
      for (int i = 0; i < S; ++i) {
        const float k = keyof<KEYS>(v[i]);
        const bool in = (k >= lo) && (k < hi);
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (m) {
          if (in) {
            const int pos = base + __popc(m & ((1u << lane) - 1u));
            sk[pos] = (static_cast<unsigned long long>(ord_bits(k)) << 32) | static_cast<unsigned>(row_of(i, jx, lane));
            sp[pos] = v[i];
          }
          base += __popc(m);
        }
      }
      __syncwarp();
      const unsigned long long mine = sk[lane];
      const float mypay = sp[lane];
      int rank = 0;
#pragma unroll
      for (int t = 0; t < 32; ++t) rank += (sk[t] < mine) ? 1 : 0;
      __syncwarp();
      if (!KEYS) {
        const unsigned ma = __ballot_sync(0xffffffffu, rank == r1 - c_lo);
        const unsigned mb = __ballot_sync(0xffffffffu, rank == r2 - c_lo);
        a = __shfl_sync(0xffffffffu, mypay, __ffs(ma) - 1);
        b = __shfl_sync(0xffffffffu, mypay, __ffs(mb) - 1);
      } else {
        const int take = r1 + 1 - c_lo;             // kept candidates = first `take` in (key,row) order
        a = warp_sum(sum_lo + ((rank < take) ? mypay : 0.f));
      }
      return;
    }
    if (iter >= 4 || !model) {
      // ---- fallback: bisect the bracket's actual extremes on the order-preserving integer image (ord_bits, with
      // -0 taken as +0 so that equal keys have one image).  The pivot is the image midpoint rounded up, so
      // vmin < p <= vmax and either side of it spans at most half the images of [vmin, vmax]: fewer than 2^32
      // images, so at most 32 such passes leave a single key, and 4 model passes + 32 + the closing one stay
      // under the 96-pass cap for any non-NaN column.  (A float midpoint removes only the top binade when the
      // bracket spans many: a column with a hundred rows one per binade ran out of passes.)
      float vmin = kInf, vmax = -kInf;
#pragma unroll
      for (int i = 0; i < S; ++i) {
        const float k = keyof<KEYS>(v[i]);
        const bool in = (k >= lo) && (k < hi);
        vmin = in ? fminf(vmin, k) : vmin;
        vmax = in ? fmaxf(vmax, k) : vmax;
      }
      vmin = warp_min_f(vmin);
      vmax = warp_max_f(vmax);
      if (!(vmin < vmax)) {
        // every element of the bracket has the same key (a tie group wider than a warp)
        if (!KEYS) { a = b = vmin; return; }
        const float part = tie_sum<S>(v, vmin, r1 + 1 - c_lo, jx, lane);
        a = warp_sum(sum_lo + part);
        return;
      }
      const uint32_t olo = ord_bits(__fadd_rn(vmin, 0.f)), ohi = ord_bits(__fadd_rn(vmax, 0.f));
      p = from_ord_bits(olo + ((ohi - olo + 1u) >> 1));
      model = false;
    }
    int c;
    float s = 0.f;
    count_pass<S, KEYS>(v, p, c, s);
    if (c <= r1) { lo = p; c_lo = c; sum_lo = s; }
    else if (c > r2) { hi = p; c_hi = c; }
    else {
      // p separates the two middle order statistics (even N median only)
      float below = -kInf, above = kInf;
#pragma unroll
      for (int i = 0; i < S; ++i) {
        below = (v[i] < p) ? fmaxf(below, v[i]) : below;
        above = (v[i] >= p) ? fminf(above, v[i]) : above;
      }
      a = warp_max_f(below);
      b = warp_min_f(above);
      return;
    }
    if (model) {
      // aim just past the target on the far side so that the next pass closes the bracket
      float step;
      if (c <= r1) { const float gap = static_cast<float>(r2 + 1 - c); step = (gap + 3.f + 0.25f * gap) / density; }
      else { const float gap = static_cast<float>(c - r1); step = -(gap + 3.f + 0.25f * gap) / density; }
      float np = p + step;
      if (!(np > lo && np < hi)) {
        if (lo > -kInf && hi < kInf) np = 0.5f * lo + 0.5f * hi;
        if (!(np > lo && np < hi)) model = false;
      }
      p = np;
    }
  }
}

// Sum, in row order, of the first `need` devs among the elements whose |dev| == T (a tie group that the
// keep boundary cuts through).  Uses ballots per slot; registers hold each 4-slot group permuted by jx.
template <int S>
__device__ __forceinline__ float tie_sum(const float (&v)[S], float T, int need, int jx, int lane) {
  float part = 0.f;
  int before = 0;
#pragma unroll
  for (int g = 0; g < S; g += 4) {
    unsigned bm[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) bm[q] = __ballot_sync(0xffffffffu, fabsf(v[g + q]) == T);
    if ((bm[0] | bm[1] | bm[2] | bm[3]) == 0u) continue;       // no member of the tie group in these 128 rows (warp-uniform)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {           // true slot order inside the group
      const int q = kk ^ jx;
      const unsigned m = q == 0 ? bm[0] : q == 1 ? bm[1] : q == 2 ? bm[2] : bm[3];
      const float val = q == 0 ? v[g] : q == 1 ? v[g + 1] : q == 2 ? v[g + 2] : v[g + 3];
      if ((m >> lane) & 1u) {
        const int rank = before + __popc(m & ((1u << lane) - 1u));
        if (rank < need) part += val;
      }
      before += __popc(m);
    }
  }
  return part;
}

// Ascending 32-lane bitonic sort of one float per lane by keyof<KEYS>() (|v| for KEYS); lanes with equal keys keep
// their own value, so nothing is duplicated or lost.  For KEYS the value is rotated left by one bit first: the
// 31 magnitude bits become the high bits and the sign the lowest, so an unsigned integer min/max orders by |v|
// (then sign) and carries the whole value along: 4 instructions per stage instead of 6 with float compares.
template <bool KEYS>
__device__ __forceinline__ float warp_sort32(float v, int lane) {
  uint32_t u = KEYS ? __funnelshift_l(__float_as_uint(v), __float_as_uint(v), 1) : 0u;
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const bool up = (k == 32) ? true : ((lane & k) == 0);
      const bool take_min = ((lane & j) == 0) == up;
      if (KEYS) {
        const uint32_t p = __shfl_xor_sync(0xffffffffu, u, j);
        u = take_min ? min(u, p) : max(u, p);
      } else {
        const float p = __shfl_xor_sync(0xffffffffu, v, j);
        v = take_min ? fminf(v, p) : fmaxf(v, p);
      }
    }
  }
  return KEYS ? __uint_as_float(__funnelshift_r(u, u, 1)) : v;
}

// One staged word as the fp32 value of the column that `sel` (unpack_sel) picks: fp32 as is; bf16 moved to the top
// half by one PRMT; fp16 moved to the bottom half by one PRMT and converted.
template <int DT>
__device__ __forceinline__ float unpack_word(uint32_t w, uint32_t sel) {
  if constexpr (DT == AFL_F32) return __uint_as_float(w);
  else if constexpr (DT == AFL_BF16) return __uint_as_float(__byte_perm(w, 0u, sel));
  else return f16_bits_to_f32(__byte_perm(w, 0u, sel));
}
template <int DT>
__device__ __forceinline__ uint32_t unpack_sel(int half) {
  if constexpr (DT == AFL_F16) return half ? 0x3232u : 0x1010u;
  else return half ? 0x3244u : 0x1044u;
}

// Where a register-resident column lives in the shared-memory tile, so that a candidate can be re-read by a
// run-time register index (a dynamic index into the register array itself would spill it to local memory).
struct ColRef {
  const uint32_t* words;     // tile word of element 0 for this lane; element i is words[(i >> 2) * 128 + (i & 3)]
  uint32_t unpack_sel;       // 16-bit formats: PRMT selector of the column's half of the word (unpack_sel<DT>)
  float med;                 // KEYS: the median that was subtracted from the registers
};
template <int DT, bool KEYS>
__device__ __forceinline__ float col_fetch(const ColRef& c, int i) {
  const uint32_t w = c.words[(i >> 2) * 128 + (i & 3)];
  const float x = unpack_word<DT>(w, c.unpack_sel);
  return KEYS ? __fsub_rn(x, c.med) : x;
}

// One element of the fused pass: below = key < a; ca += below; (KEYS) sa += below ? v : 0; inmask |= bit when
// a <= key < b.  Written in PTX so that it stays 4 (5) instructions: the C++ form was compiled to 14 per element
// (the count became a set/clear bit mask, and the list address was rebuilt under every store's predicate).
template <bool KEYS>
__device__ __forceinline__ void fused_step(float v, float a, float b, uint32_t bit, int& ca, uint32_t& inmask, float& sa) {
  if (KEYS) {
    asm("{\n\t.reg .pred p, q;\n\t.reg .f32 k;\n\t"
        "abs.f32 k, %3;\n\t"
        "setp.lt.f32 p, k, %4;\n\t"
        "setp.lt.and.f32 q, k, %5, !p;\n\t"
        "@p add.s32 %0, %0, 1;\n\t"
        "@p add.rn.f32 %2, %2, %3;\n\t"
        "@q or.b32 %1, %1, %6;\n\t}"
        : "+r"(ca), "+r"(inmask), "+f"(sa)
        : "f"(v), "f"(a), "f"(b), "r"(bit));
  } else {
    asm("{\n\t.reg .pred p, q;\n\t"
        "setp.lt.f32 p, %2, %3;\n\t"
        "setp.lt.and.f32 q, %2, %4, !p;\n\t"
        "@p add.s32 %0, %0, 1;\n\t"
        "@q or.b32 %1, %1, %5;\n\t}"
        : "+r"(ca), "+r"(inmask)
        : "f"(v), "f"(a), "f"(b), "r"(bit));
  }
}

// Fast path.  One fused pass over the registers with a model bracket [a, b): counts #{key < a} (and the
// lane-local dev sum below a) and marks the in-bracket elements in a per-lane bit mask (no stores, no ballots,
// no branches).  If the target rank(s) fall inside and <= 32 candidates were marked, each lane re-reads its
// few candidates from the tile into a dense 32-entry list (exclusive prefix of the per-lane counts), and the
// list is sorted with a 15-stage shuffle network.  Returns false (state updated: lo/c_lo/sum_lo or hi/c_hi
// tightened where the pass proved a bound) when the general path has to take over.
template <int S, bool KEYS, int DT>
__device__ __forceinline__ bool select_fast(const float (&v)[S], const ColRef& col, int n, int r1, int r2, float p0,
                                            float density, int lane, int jx, uint32_t* scratch, float& lo, float& hi,
                                            int& c_lo, int& c_hi, float& sum_lo, float& out_a, float& out_b) {
  static_assert(S <= 32, "one mask bit per register-resident element");
  if (!((density > 0.f) && (density < kInf) && (p0 == p0) && (fabsf(p0) < kInf))) return false;
  float center = p0;
  const float inv_density = __fdividef(1.f, density);       // model only: approximate division is enough
  float halfw = (11.f + 0.5f * static_cast<float>(r2 - r1)) * inv_density;
#pragma unroll 1
  for (int attempt = 0; attempt < 3; ++attempt) {
    float a = center - halfw, b = center + halfw;
    if (KEYS && a < 0.f) a = 0.f;
    if (!(a > lo)) a = lo;
    if (!(b < hi)) b = hi;
    if (!(a < b)) return false;
    int ca = 0;
    float sa = 0.f;
    uint32_t inmask = 0u;
#pragma unroll
    for (int i = 0; i < S; ++i) fused_step<KEYS>(v[i], a, b, 1u << i, ca, inmask, sa);
    const int mine = __popc(inmask);
    const int c_a = warp_sum_i(ca);
    const int cin = warp_sum_i(mine);
    const int c_b = c_a + cin;
    const bool inside = (c_a <= r1) && (r2 < c_b);
    if (inside && cin <= 32) {
      // ---- dense compaction: exclusive prefix of the per-lane counts, then one candidate per lane
      int incl = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      float* dense = reinterpret_cast<float*>(scratch);              // [32]
      int pos = incl - mine;
      for (uint32_t m = inmask; m != 0u; m &= m - 1u) dense[pos++] = col_fetch<DT, KEYS>(col, __ffs(m) - 1);
      __syncwarp();
      const bool have = lane < cin;
      const float val = have ? dense[lane] : kInf;
      __syncwarp();
      // 15-stage shuffle bitonic sort of the (<= 32) candidates by key; equal keys may end up in any order, which
      // is fine: for the median equal keys are equal values, for the |dev| threshold a tie group that the keep
      // boundary cuts is resolved in row order by tie_sum() on the register-resident column, not on these lanes.
      // (round 1 ranked every candidate against every other: 31 shuffles + 93 ALU ops, 21 % of the kernel.)
      const float sv = warp_sort32<KEYS>(val, lane);
      if (!KEYS) {
        out_a = __shfl_sync(0xffffffffu, sv, r1 - c_a);
        out_b = __shfl_sync(0xffffffffu, sv, r2 - c_a);
        return true;
      }
      const float skey = fabsf(sv);
      const int take = r1 + 1 - c_a;            // number of candidates kept, in (key, row) order
      const float T = __shfl_sync(0xffffffffu, skey, take - 1);                  // the boundary candidate's key
      const int n_less = __popc(__ballot_sync(0xffffffffu, have && skey < T));
      const int group = __popc(__ballot_sync(0xffffffffu, have && skey == T));
      const int need = take - n_less;
      float part = sa + ((have && skey < T) ? sv : 0.f);
      if (need == group) part += (have && skey == T) ? sv : 0.f;    // whole tie group kept: order irrelevant
      else part += tie_sum<S>(v, T, need, jx, lane);                   // boundary cuts the group: row order
      out_a = warp_sum(part);
      return true;
    }
    if (!KEYS && c_a > r1 && c_a <= r2) {
      // the lower pivot separates the two middle order statistics (even N): read them off directly
      float below = -kInf, above = kInf;
#pragma unroll
      for (int i = 0; i < S; ++i) {
        below = (v[i] < a) ? fmaxf(below, v[i]) : below;
        above = (v[i] >= a) ? fminf(above, v[i]) : above;
      }
      out_a = warp_max_f(below);
      out_b = warp_min_f(above);
      return true;
    }
    // ---- not closed: keep what the pass proved (invariants: c_lo <= r1, r2 < c_hi) and aim again
    const float mid = 0.5f * static_cast<float>(r1 + r2) + 0.5f;
    if (c_a <= r1) { lo = a; c_lo = c_a; sum_lo = sa; } else { hi = a; c_hi = c_a; }
    if (c_b > r2 && b < hi) { hi = b; c_hi = c_b; }
    if (inside) {                                   // too many candidates: shrink around the interpolated rank
      const float w = __fdividef(b - a, static_cast<float>(cin > 0 ? cin : 1));
      center = a + (mid - static_cast<float>(c_a)) * w;
      halfw = 9.f * w;
    } else if (c_a > r2) {                          // target below the bracket
      center = a - (static_cast<float>(c_a) - mid) * inv_density;
      halfw = (5.f + 0.35f * (static_cast<float>(c_a) - mid)) * inv_density;
    } else {                                        // target above the bracket
      center = b + (mid - static_cast<float>(c_b)) * inv_density;
      halfw = (5.f + 0.35f * (mid - static_cast<float>(c_b))) * inv_density;
    }
  }
  return false;
}

// ---------------- staging: coalesced 16-byte row-segment loads -> swizzled smem ----------------
// Thread t loads the 16-byte chunk j = t&3 of row (it*64 + t>>2) in iteration `it`.  Row r lives in
// slot r>>5 of lane r&31; slot-group m = slot>>2 and the XOR-ed slot position are compile-time
// functions of `it`, so every store below has an immediate offset from one of two per-thread bases.
// The problem a CTA works on: blockIdx.y, or for a class launch (CLASS) the class's blockIdx.y-th problem.
template <bool CLASS>
__device__ __forceinline__ unsigned problem_of(const Params& P) {
  if constexpr (CLASS) return static_cast<unsigned>(static_cast<const ClassParams&>(P).perm[blockIdx.y]);
  else return blockIdx.y;
}

// The tile of one problem: its matrix at `base`, its row_index (may be NULL) and its participating rows sh.n_rows.
template <int S, int DT>
__device__ __forceinline__ void stage_rows(const Params& P, const TmShape& sh, uint32_t* tile, int64_t col0,
                                           const uint8_t* base, const int* row_index) {
  constexpr int kGroups = S / 4;
  constexpr bool W16 = DT != AFL_F32;                   // two 16-bit columns per word
  const int tid = threadIdx.x;
  const int es = W16 ? 2 : 4;
  const int cols_per_tile = W16 ? 32 : 16;
  const uint32_t sentinel = DT == AFL_F16 ? 0x7C007C00u : DT == AFL_BF16 ? 0x7F807F80u : 0x7F800000u;   // +inf
  constexpr int kIters = (32 * S * 4) / kThreads;      // S/2
  const bool full_tile = P.vec_ok && (col0 + cols_per_tile <= P.d);
  const int rowq = tid >> 2, j = tid & 3, l = rowq & 31, hi2 = tid >> 7;
  uint32_t* b0 = tile + (4 * j * kGroups) * 128 + l * 4 + (hi2 ^ j);
  uint32_t* b1 = tile + (4 * j * kGroups) * 128 + l * 4 + ((2 + hi2) ^ j);
  const int64_t c = col0 + static_cast<int64_t>(j) * (16 / es);
  if (full_tile) {
    // every 16-byte load of the tile is issued before the first store: one DRAM round trip per CTA instead of
    // one per batch of four (the kernel has the registers: the per-column code needs 80 anyway), and ~8
    // instructions per load so that the whole path stays a few hundred bytes of code
    // (branch-free: rows past n_rows re-read the last row and are replaced by the sentinel at the store)
    int gr[kIters];
    const int last = sh.n_rows - 1;
    if (row_index) {
#pragma unroll
      for (int it = 0; it < kIters; ++it) gr[it] = row_index[min(it * 64 + rowq, last)];
#pragma unroll
      for (int it = 0; it < kIters; ++it) gr[it] = gr[it] < 0 ? gr[it] + P.n_total : gr[it];
    } else {
#pragma unroll
      for (int it = 0; it < kIters; ++it) gr[it] = min(it * 64 + rowq, last);
    }
    const uint8_t* colbase = base + c * es;
    const int64_t row_bytes = P.ld * es;
    uint4 val[kIters];
#pragma unroll
    for (int it = 0; it < kIters; ++it)
      val[it] = ldg_stream_u4(reinterpret_cast<const uint4*>(colbase + gr[it] * row_bytes));
#pragma unroll
    for (int it = 0; it < kIters; ++it) {
      const bool pad = it * 64 + rowq > last;
      uint32_t* b = (it & 1) ? b1 : b0;
      const int m = it >> 1;
      b[(0 * kGroups + m) * 128] = pad ? sentinel : val[it].x;
      b[(1 * kGroups + m) * 128] = pad ? sentinel : val[it].y;
      b[(2 * kGroups + m) * 128] = pad ? sentinel : val[it].z;
      b[(3 * kGroups + m) * 128] = pad ? sentinel : val[it].w;
    }
    return;
  }
  // ragged last tile / unaligned matrix: element-wise, one rolled iteration at a time (cold: keep the code small)
#pragma unroll 1
  for (int it = 0; it < kIters; ++it) {
    const int r = it * 64 + rowq;
    uint32_t w[4] = {sentinel, sentinel, sentinel, sentinel};
    if (r < sh.n_rows) {
      int gr = row_index ? row_index[r] : r;
      gr = gr < 0 ? gr + P.n_total : gr;
      const uint8_t* src = base + (static_cast<int64_t>(gr) * P.ld + c) * es;
      w[0] = w[1] = w[2] = w[3] = 0u;
      if (W16) {
        const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (c + e < P.d) w[e >> 1] |= static_cast<uint32_t>(s16[e]) << ((e & 1) * 16);
      } else {
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (c + e < P.d) w[e] = s32[e];
      }
    }
    uint32_t* b = ((it & 1) ? b1 : b0) + (it >> 1) * 128;
    b[(0 * kGroups) * 128] = w[0];
    b[(1 * kGroups) * 128] = w[1];
    b[(2 * kGroups) * 128] = w[2];
    b[(3 * kGroups) * 128] = w[3];
  }
}

template <int S, int DT, bool CLASS>
__device__ __forceinline__ void stage_tile(const Params& P, const TmShape& sh, uint32_t* tile, int64_t col0) {
  const int es = DT != AFL_F32 ? 2 : 4;
  const uint8_t* base;
  const int* row_index;
  if constexpr (CLASS) {
    const int64_t b = problem_of<CLASS>(P);
    base = static_cast<const uint8_t*>(P.G) + b * P.g_batch * es;
    row_index = P.row_index ? P.row_index + b * P.ri_batch : nullptr;
  } else {
    base = static_cast<const uint8_t*>(P.G) + static_cast<int64_t>(blockIdx.y) * P.g_batch * es;
    row_index = P.row_index ? P.row_index + static_cast<int64_t>(blockIdx.y) * P.ri_batch : nullptr;
  }
  stage_rows<S, DT>(P, sh, tile, col0, base, row_index);
}

// ---------------- general per-column path (any data): one warp, one column ----------------
// `half` selects the 16-bit column inside the 32-bit word-column cw (ignored for fp32).
template <int S, int DT>
__device__ __forceinline__ float general_column_impl(const TmShape& P, const uint32_t* tile, int cw, int half,
                                                     uint32_t* scratch, int lane) {
  constexpr int kGroups = S / 4;
  const int n = P.n_rows;
  const float fn = static_cast<float>(n);
  const int jx = (cw >> 2) & 3;
  const uint4* t4 = reinterpret_cast<const uint4*>(tile) + (cw * kGroups) * 32 + lane;
  // 16-bit -> fp32 is one PRMT with a run-time selector (`half` is a loop variable: a ?: costs two predicated
  // instructions), plus the conversion for fp16
  const uint32_t sel = unpack_sel<DT>(half);
  ColRef col{reinterpret_cast<const uint32_t*>(t4), sel, 0.f};
  float x[S];
#pragma unroll
  for (int m = 0; m < kGroups; ++m) {
    const uint4 t = t4[m * 32];
    const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) x[4 * m + q] = unpack_word<DT>(w[q], sel);
  }

  // mean / sigma of the column (pivot model only; never enters the result).  The kernel is instantiated with
  // 16 * S < n_rows <= 32 * S (S >= 8), so the first half of the slot groups holds real rows only; in the second half a
  // padded row is +inf and is skipped by predicate (no branches: the warp-uniform "is this group full" tests of
  // round 1 cost an instruction-fetch bubble each).
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < S; ++i) {
    if (S >= 8 && i < S / 2) {             // the launcher picks S with 32 * 4 * ceil(S / 8) <= n_rows for S >= 8
      s1 += x[i]; s2 = fmaf(x[i], x[i], s2);
    } else {
      asm("{\n\t.reg .pred p;\n\t"
          "setp.lt.f32 p, %2, 0f7F800000;\n\t"
          "@p add.rn.f32 %0, %0, %2;\n\t"
          "@p fma.rn.f32 %1, %2, %2, %1;\n\t}"
          : "+f"(s1), "+f"(s2) : "f"(x[i]));
    }
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  const float mean = __fdividef(s1, fn);
  const float var = fmaxf(__fdividef(s2, fn) - mean * mean, 0.f);
  const float inv_sd = rsqrtf(var);              // var == 0: +inf -> the densities below fail the model test
  const float sd = var * inv_sd;                 // (NaN for var == 0: same effect on the |dev| pivot)

  // median (np.median: even N -> mean of the two middle order statistics, fp32)
  float a, b;
  {
    float lo = -kInf, hi = kInf, sl = 0.f;
    int c_lo = 0, c_hi = n;
    if (!select_fast<S, false, DT>(x, col, n, (n - 1) >> 1, n >> 1, mean, P.med_density * inv_sd, lane, jx, scratch, lo, hi, c_lo,
                               c_hi, sl, a, b))
      warp_select<S, false>(x, n, (n - 1) >> 1, n >> 1, mean, P.med_density * inv_sd, lane, jx, scratch, lo, hi, c_lo,
                            c_hi, 0.f, a, b);
  }
  const float med = ((n & 1) != 0) ? a : __fdiv_rn(__fadd_rn(a, b), 2.0f);

  float res;
  if (P.keep <= 0) {
    res = __int_as_float(0x7fc00000);           // np.mean([]) is nan
  } else {
#pragma unroll
    for (int i = 0; i < S; ++i) x[i] = __fsub_rn(x[i], med);      // devs; padded rows stay +inf
    float total, unused;
    float lo = -kInf, hi = kInf, sl = 0.f;
    int c_lo = 0, c_hi = n;
    col.med = med;
    if (!select_fast<S, true, DT>(x, col, n, P.keep - 1, P.keep - 1, P.key_q * sd, P.key_density * inv_sd, lane, jx, scratch, lo, hi,
                              c_lo, c_hi, sl, total, unused)) {
      // General path.  Infinite deviations (an inf in the column, or fl32(x - med) overflowing) share the key +inf with
      // the padded rows, so the bracket's upper count is the number of finite keys, not n.  When the keep boundary is
      // at or past it, the threshold is +inf: every finite deviation is kept, and the infinite ones in row order
      // (padded rows come after every real row, so tie_sum never reaches them).
      int c_fin;
      float s_fin = 0.f;
      count_pass<S, true>(x, kInf, c_fin, s_fin);
      if (P.keep > c_fin) {
        total = warp_sum(s_fin + tie_sum<S>(x, kInf, P.keep - c_fin, jx, lane));
      } else {
        if (hi == kInf) c_hi = c_fin;
        warp_select<S, true>(x, n, P.keep - 1, P.keep - 1, P.key_q * sd, P.key_density * inv_sd, lane, jx, scratch, lo, hi,
                             c_lo, c_hi, sl, total, unused);
      }
    }
    res = __fadd_rn(__fdiv_rn(total, static_cast<float>(P.keep)), med);
  }
  return res;
}

constexpr int kScratchWords = 96;              // per warp: dense candidate list [32] (fast path) / (key,row) u64[32] + payload[32] (general path)

// S <= 20 (up to 640 rows: Bulyan's second stage at N = 500 and N = 1000) leaves room for four CTAs per SM in shared memory; ask
// the compiler for 64 registers there (resident warps are what hides the shuffle chains of the scans and sorts).
// EACH: problem blockIdx.y's constants come from the per-problem table P.each (batches only).  A separate instance:
// holding them in registers instead of reading the constant bank takes the fp32 kernel from 48 to 54 registers, which
// would cost the single calls a fifth CTA per SM.  CLASS (with EACH): a class launch, problem P.perm[blockIdx.y].
// The class instances hold the table constants and the problem index in registers too: they would spill from S = 16 on
// at the single calls' bounds, so they ask for fewer CTAs per SM: 3 at S = 16 (80 registers), 2 from S = 20 (128; the
// 16-bit S = 20 instances still spill at 80).
template <int S, int DT, bool EACH, bool CLASS = false>
__global__ void __launch_bounds__(kThreads, CLASS ? (S <= 12 ? 4 : S <= 16 ? 3 : 2)
                                                  : (S <= 20 ? 4 : 3))      // (S = 24 fits 4 CTAs in shared memory too, but the fp32 instance spills at 64 registers)
trimmed_mean_kernel(const KernelParams<CLASS> P) {
  static_assert(EACH || !CLASS, "a class launch reads the table");
  extern __shared__ __align__(1024) uint32_t tile[];     // [16 word-cols][S/4 groups][32 lanes][4 slots] + scratch
  constexpr int kGroups = S / 4;
  constexpr bool W16 = DT != AFL_F32;                    // bf16 / fp16: two columns per word-column
  const int tid = threadIdx.x, warp = tid >> 5;
  const int cols_per_tile = W16 ? 32 : 16;
  const int64_t col0 = static_cast<int64_t>(blockIdx.x) * cols_per_tile;
  TmShape sh = P.tm;
  if constexpr (CLASS) sh = P.each[problem_of<CLASS>(P)].tm;
  else if constexpr (EACH) sh = P.each[blockIdx.y].tm;
  stage_tile<S, DT, CLASS>(P, sh, tile, col0);
  // read once, after staging: `volatile` keeps ptxas from re-reading the special register (S2R, ~50 cycles of
  // latency) in front of every scan and sort of the per-column code to save one register
  int lane = tid & 31, warp_o = warp;
  if (W16 || S < 32) {        // (the fp32 S = 32 instance is at the 80-register limit: there it would only add spills)
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    asm volatile("mov.u32 %0, %1;" : "=r"(warp_o) : "r"(warp));
  }
  __syncthreads();
  uint32_t* scratch = tile + kWordCols * kGroups * 128 + warp_o * kScratchWords;
#pragma unroll 1
  for (int cw = warp_o; cw < kWordCols; cw += kWarps) {
#pragma unroll 1
    for (int half = 0; half < (W16 ? 2 : 1); ++half) {
      const int64_t col = col0 + (W16 ? 2 * cw + half : cw);
      if (col >= P.d) break;                         // warp-uniform
      const float res = general_column_impl<S, DT>(sh, tile, cw, half, scratch, lane);
      if constexpr (CLASS) {
        if (lane == 0) P.out[static_cast<int64_t>(problem_of<CLASS>(P)) * P.out_batch + col] = res;
      } else {
        if (lane == 0) P.out[static_cast<int64_t>(blockIdx.y) * P.out_batch + col] = res;
      }
    }
  }
}

// A device-count class launch's arguments (trimmed_mean_dev_kernel): Params, and the class's problems perm[start[cls] ..
// start[cls + 1]), device values that class_perm_kernel (capi.cu) wrote.
struct DevClassParams : Params {
  const int* perm;
  const int* start;       // kSlotClasses + 1 offsets into perm
  int cls, batch;
  int tiles;              // column tiles per problem, < 2^31
  int step_p, step_t;     // gridDim.x as (problems, tiles): gridDim.x = step_p * tiles + step_t
};

// Device-count class launch: a persistent grid whose size the host knows without the class's size strides over the
// class's work items i in [0, count * tiles), item i being problem perm[start[cls] + i / tiles] and column tile
// i % tiles.  So the launch needs no class size on the host, and an absent class costs one wave of CTAs that read a
// zero count.  Per column it runs the CLASS instance's stage_rows and general_column_impl with the same S, so a
// column's result does not depend on which CTA computed it: the outputs are the host-count launch's bit for bit.
// Launch bounds: the CLASS instances' for fp32.  The 16-bit instances spill at those (the per-item loop keeps a few
// more values live than a CLASS CTA's single problem), so they ask for fewer CTAs per SM from S = 8 on: 80 registers
// at S = 8, 128 at S = 12 to 24, and one CTA per SM at S = 28 and 32.
template <int DT, int S>
constexpr int dev_min_ctas() {
  if (DT == AFL_F32) return S <= 12 ? 4 : S <= 16 ? 3 : 2;
  return S <= 4 ? 4 : S <= 8 ? 3 : S <= 24 ? 2 : 1;
}
template <int S, int DT>
__global__ void __launch_bounds__(kThreads, dev_min_ctas<DT, S>())
trimmed_mean_dev_kernel(const DevClassParams P) {
  extern __shared__ __align__(1024) uint32_t tile[];     // trimmed_mean_kernel's layout
  constexpr int kGroups = S / 4;
  constexpr bool W16 = DT != AFL_F32;
  const int es = W16 ? 2 : 4;
  const int cols_per_tile = W16 ? 32 : 16;
  const int tid = threadIdx.x, warp = tid >> 5;
  // The item (p, t) = (i / tiles, i % tiles) and the class's span live in shared memory: the column code needs every
  // register it had in the CLASS instance, and loop state held in registers across it made the 16-bit instances
  // spill.  Thread 0 writes the next item into the other slot of `item`; the barrier at the end of an item orders
  // that write before every read of it, and after every read of the slot's previous contents.
  __shared__ int item[2][2];
  __shared__ int span[2];                              // first, count: the offsets clamped to [0, batch]
  if (tid == 0) {
    const int first = min(max(P.start[P.cls], 0), P.batch);
    span[0] = first;
    span[1] = min(max(P.start[P.cls + 1], first), P.batch) - first;
    item[0][0] = static_cast<int>(blockIdx.x / static_cast<unsigned>(P.tiles));
    item[0][1] = static_cast<int>(blockIdx.x % static_cast<unsigned>(P.tiles));
  }
  __syncthreads();
#pragma unroll 1
  for (int k = 0;; k ^= 1) {
    const int p = item[k][0], t = item[k][1];
    if (p >= span[1]) break;                         // CTA-uniform; p grows every item, so the loop ends
    if (tid == 0) {                                  // i + gridDim.x without a division
      unsigned nt = static_cast<unsigned>(t) + P.step_t;
      int np = p + P.step_p;
      if (nt >= static_cast<unsigned>(P.tiles)) { nt -= P.tiles; ++np; }
      item[k ^ 1][0] = np;
      item[k ^ 1][1] = static_cast<int>(nt);
    }
    const int64_t b = P.perm[span[0] + p];
    const int64_t col0 = static_cast<int64_t>(t) * cols_per_tile;
    const TmShape sh = P.each[b].tm;
    stage_rows<S, DT>(P, sh, tile, col0, static_cast<const uint8_t*>(P.G) + b * P.g_batch * es,
                      P.row_index ? P.row_index + b * P.ri_batch : nullptr);
    int lane = tid & 31, warp_o = warp;
    if (W16 || S < 32) {      // as trimmed_mean_kernel
      asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
      asm volatile("mov.u32 %0, %1;" : "=r"(warp_o) : "r"(warp));
    }
    __syncthreads();
    uint32_t* scratch = tile + kWordCols * kGroups * 128 + warp_o * kScratchWords;
#pragma unroll 1
    for (int cw = warp_o; cw < kWordCols; cw += kWarps) {
#pragma unroll 1
      for (int half = 0; half < (W16 ? 2 : 1); ++half) {
        const int64_t col = col0 + (W16 ? 2 * cw + half : cw);
        if (col >= P.d) break;                         // warp-uniform
        const float res = general_column_impl<S, DT>(sh, tile, cw, half, scratch, lane);
        if (lane == 0) P.out[b * P.out_batch + col] = res;
      }
    }
    __syncthreads();          // every warp is done with the tile before the next item re-stages it
  }
}

// ---------------- more than 1024 participating rows: shared-memory bisection kernel (any n that fits) ----------------
// The register-resident kernels above hold ceil(n/32) <= 32 values per lane.  Beyond that a CTA stages a 16-byte-wide
// column strip of ALL rows in shared memory ([row][4 words], up to kLargeMaxRows rows) and one warp per column finds
// the order statistics by bisection on the order-preserving integer image of the values (32 counting passes over
// shared memory per statistic), then the |dev| threshold the same way, and resolves a tie group at the threshold in row
// order with ballots.  Exact for any data; slow (a fallback: the reference has no client-count limit, defences.py:44-52).
constexpr int kLargeMaxRows = 12288;          // 12288 rows x 16 B = 192 KB of shared memory

// w16: 16-bit elements, two per word (bf16, or fp16 when F16)
template <bool F16>
__device__ __forceinline__ float strip_value(const uint32_t* strip, int row, int col_in_strip, bool w16) {
  if (!w16) return __uint_as_float(strip[row * 4 + col_in_strip]);
  const uint32_t w = strip[row * 4 + (col_in_strip >> 1)];
  if (F16) return f16_bits_to_f32((col_in_strip & 1) ? (w >> 16) : w);
  return __uint_as_float((col_in_strip & 1) ? (w & 0xFFFF0000u) : (w << 16));
}

// k-th smallest (0-based) key among this warp's column, keys = ord_bits(f(value)); F = 0: value, F = 1: |fl32(value - med)|
template <int F, bool F16>
__device__ __forceinline__ uint32_t warp_kth_key(const uint32_t* strip, int n, int cis, bool w16, float med, int k, int lane) {
  uint32_t lo = 0u, hi = 0xFFFFFFFFu;                      // invariant: count(key < lo) <= k < count(key <= hi)
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    int c = 0;
    for (int r = lane; r < n; r += 32) {
      float v = strip_value<F16>(strip, r, cis, w16);
      if (F) v = fabsf(__fsub_rn(v, med));
      c += (ord_bits(v) <= mid) ? 1 : 0;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if (c > k) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// bf16 != 0: 16-bit elements (bf16, or fp16 in the F16 instance)
template <bool F16>
__global__ void __launch_bounds__(256, 1)
trimmed_mean_large_kernel(const Params P, int bf16) {
  extern __shared__ __align__(16) uint32_t strip[];        // [n_rows][4 words]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = P.tm.n_rows;
  const int es = bf16 ? 2 : 4;
  const int cols = bf16 ? 8 : 4;
  const int64_t col0 = static_cast<int64_t>(blockIdx.x) * cols;
  const uint8_t* base = static_cast<const uint8_t*>(P.G) + static_cast<int64_t>(blockIdx.y) * P.g_batch * es;
  const int* row_index = P.row_index ? P.row_index + static_cast<int64_t>(blockIdx.y) * P.ri_batch : nullptr;
  for (int r = tid; r < n; r += blockDim.x) {
    int gr = row_index ? row_index[r] : r;
    gr = gr < 0 ? gr + P.n_total : gr;
    const uint8_t* src = base + (static_cast<int64_t>(gr) * P.ld + col0) * es;
    uint32_t w[4] = {0u, 0u, 0u, 0u};
    if (P.vec_ok && col0 + cols <= P.d) {
      const uint4 t = ldg_stream_u4(reinterpret_cast<const uint4*>(src));
      w[0] = t.x; w[1] = t.y; w[2] = t.z; w[3] = t.w;
    } else if (bf16) {
      const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
      for (int e = 0; e < 8; ++e)
        if (col0 + e < P.d) w[e >> 1] |= static_cast<uint32_t>(s16[e]) << ((e & 1) * 16);
    } else {
      const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
      for (int e = 0; e < 4; ++e)
        if (col0 + e < P.d) w[e] = s32[e];
    }
    *reinterpret_cast<uint4*>(strip + r * 4) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  __syncthreads();
  for (int cis = warp; cis < cols; cis += 8) {
    const int64_t col = col0 + cis;
    if (col >= P.d) break;
    const float a = from_ord_bits(warp_kth_key<0, F16>(strip, n, cis, bf16 != 0, 0.f, (n - 1) >> 1, lane));
    const float b = (n & 1) ? a : from_ord_bits(warp_kth_key<0, F16>(strip, n, cis, bf16 != 0, 0.f, n >> 1, lane));
    const float med = (n & 1) ? a : __fdiv_rn(__fadd_rn(a, b), 2.0f);
    float res;
    if (P.tm.keep <= 0) {
      res = __int_as_float(0x7fc00000);
    } else {
      const uint32_t To = warp_kth_key<1, F16>(strip, n, cis, bf16 != 0, med, P.tm.keep - 1, lane);   // threshold key (as ord bits)
      // sum of the devs strictly below the threshold, then the first `need` of the tie group in row order
      float part = 0.f;
      int below = 0;
      for (int r = lane; r < n; r += 32) {
        const float dv = __fsub_rn(strip_value<F16>(strip, r, cis, bf16 != 0), med);
        const bool lt = ord_bits(fabsf(dv)) < To;
        part += lt ? dv : 0.f;
        below += lt ? 1 : 0;
      }
      below = __reduce_add_sync(0xffffffffu, below);
      int need = P.tm.keep - below;
      for (int r0 = 0; r0 < n && need > 0; r0 += 32) {       // rows in order: r0 .. r0+31 <-> lanes 0..31
        const int r = r0 + lane;
        float dv = 0.f;
        bool tie = false;
        if (r < n) { dv = __fsub_rn(strip_value<F16>(strip, r, cis, bf16 != 0), med); tie = ord_bits(fabsf(dv)) == To; }
        const unsigned m = __ballot_sync(0xffffffffu, tie);
        if (tie && __popc(m & ((1u << lane) - 1u)) < need) part += dv;
        need -= __popc(m);
      }
      const float total = warp_sum(part);
      res = __fadd_rn(__fdiv_rn(total, static_cast<float>(P.tm.keep)), med);
    }
    if (lane == 0) P.out[static_cast<int64_t>(blockIdx.y) * P.out_batch + col] = res;
  }
}

// perm != NULL: a class launch over `batch` problems perm[0 .. batch) (trimmed_mean_classes)
template <int S>
static int launch(const Params& P, int dtype, int batch, cudaStream_t stream, const int* perm = nullptr) {
  const size_t smem = static_cast<size_t>(S) * 2048 + kWarps * kScratchWords * 4;
  const int cols = dtype != AFL_F32 ? 32 : 16;
  const dim3 grid(static_cast<unsigned>(ceil_div64(P.d, cols)), batch);
  ProfScope ps("trimmed_mean", stream);
  auto go = [&](auto kernel, const auto& args) -> int {
    AFL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    kernel<<<grid, kThreads, smem, stream>>>(args);
    AFL_LAUNCH_CHECK("trimmed_mean_kernel");
    return AFL_OK;
  };
  if (perm) {
    ClassParams C{};
    static_cast<Params&>(C) = P;
    C.perm = perm;
    return dtype == AFL_BF16  ? go(trimmed_mean_kernel<S, AFL_BF16, true, true>, C)
           : dtype == AFL_F16 ? go(trimmed_mean_kernel<S, AFL_F16, true, true>, C)
                              : go(trimmed_mean_kernel<S, AFL_F32, true, true>, C);
  }
  if constexpr (S == 4) {
    if (P.each)
      return dtype == AFL_BF16  ? go(trimmed_mean_kernel<S, AFL_BF16, true>, P)
             : dtype == AFL_F16 ? go(trimmed_mean_kernel<S, AFL_F16, true>, P)
                                : go(trimmed_mean_kernel<S, AFL_F32, true>, P);
  }
  return dtype == AFL_BF16  ? go(trimmed_mean_kernel<S, AFL_BF16, false>, P)
         : dtype == AFL_F16 ? go(trimmed_mean_kernel<S, AFL_F16, false>, P)
                            : go(trimmed_mean_kernel<S, AFL_F32, false>, P);
}

// One device-count class launch (trimmed_mean_dev_kernel) of class cls over a batch of `batch` problems.  Grid:
// min(resident CTAs of the instance x SMs, tiles x batch), the occupancy cached per device and instance.
template <int S>
static int launch_dev(const Params& P, int dtype, int batch, cudaStream_t stream, const int* perm, const int* start,
                      int cls) {
  const size_t smem = static_cast<size_t>(S) * 2048 + kWarps * kScratchWords * 4;
  const int cols = dtype != AFL_F32 ? 32 : 16;
  const int64_t tiles = ceil_div64(P.d, cols);
  if (tiles > INT32_MAX) { set_error("afl_trimmed_mean: d = %lld is too wide", static_cast<long long>(P.d)); return AFL_ERR_UNSUPPORTED; }
  DevClassParams C{};
  static_cast<Params&>(C) = P;
  C.perm = perm; C.start = start; C.cls = cls; C.batch = batch; C.tiles = static_cast<int>(tiles);
  ProfScope ps("trimmed_mean", stream);
  auto go = [&](auto kernel, int (&smem_done)[kMaxDevices], int (&resident)[kMaxDevices]) -> int {
    AFL_CUDA(ensure_dyn_smem(kernel, static_cast<int>(smem), smem_done));
    const int dev = current_device();
    if (!resident[dev]) {
      int r = 0;
      AFL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r, kernel, kThreads, smem));
      resident[dev] = r > 0 ? r : 1;
    }
    const int64_t work = tiles * batch, wave = static_cast<int64_t>(resident[dev]) * sm_count();
    const int grid = static_cast<int>(work < wave ? work : wave);
    C.step_p = grid / C.tiles;
    C.step_t = grid % C.tiles;
    kernel<<<grid, kThreads, smem, stream>>>(C);
    AFL_LAUNCH_CHECK("trimmed_mean_dev_kernel");
    return AFL_OK;
  };
  static int smem_done[3][kMaxDevices], resident[3][kMaxDevices];
  return dtype == AFL_BF16  ? go(trimmed_mean_dev_kernel<S, AFL_BF16>, smem_done[1], resident[1])
         : dtype == AFL_F16 ? go(trimmed_mean_dev_kernel<S, AFL_F16>, smem_done[2], resident[2])
                            : go(trimmed_mean_dev_kernel<S, AFL_F32>, smem_done[0], resident[0]);
}

// `batch` problems (grid y): problem b reads G + b * g_batch and row_index + b * ri_batch, and writes out + b * out_batch.
// each (device, may be NULL; n_rows <= 128): problem b's participating rows and constants are each[b].tm, at most n_rows.
int trimmed_mean_batched(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                         int corrupted_count, float* out, int batch, int64_t g_batch, int ri_batch, int64_t out_batch,
                         cudaStream_t stream, const ProblemParams* each) {
  if (!G || !out || n < 1 || d < 1 || ld < d || n_rows < 1) { set_error("afl_trimmed_mean: bad argument"); return AFL_ERR_BAD_ARG; }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_trimmed_mean: dtype"); return AFL_ERR_UNSUPPORTED; }
  if (n_rows > kLargeMaxRows) {
    set_error("afl_trimmed_mean: at most %d participating rows fit the shared-memory strip (got %d)", kLargeMaxRows, n_rows);
    return AFL_ERR_UNSUPPORTED;
  }
  if (each && n_rows > 128) { set_error("afl_trimmed_mean: a per-problem table needs n_rows <= 128"); return AFL_ERR_UNSUPPORTED; }
  Params P{};
  P.G = G; P.row_index = row_index; P.out = out; P.d = d; P.ld = ld; P.n_total = n; P.tm = shape(n_rows, corrupted_count);
  P.each = each; P.g_batch = g_batch; P.out_batch = out_batch; P.ri_batch = ri_batch;
  const int64_t es = dtype == AFL_F32 ? 4 : 2;
  P.vec_ok = (reinterpret_cast<uintptr_t>(G) % 16 == 0) && ((ld * es) % 16 == 0) && (batch == 1 || (g_batch * es) % 16 == 0);
  if (n_rows > 1024) {
    const size_t smem = static_cast<size_t>(n_rows) * 16;
    const int cols = dtype != AFL_F32 ? 8 : 4;
    const dim3 grid(static_cast<unsigned>(ceil_div64(d, cols)), batch);
    static int smem_attr_done[kMaxDevices] = {0}, smem_attr_done_f16[kMaxDevices] = {0};
    ProfScope ps("trimmed_mean", stream);
    if (dtype == AFL_F16) {
      AFL_CUDA(ensure_dyn_smem(trimmed_mean_large_kernel<true>, static_cast<int>(kLargeMaxRows) * 16, smem_attr_done_f16));
      trimmed_mean_large_kernel<true><<<grid, 256, smem, stream>>>(P, 1);
    } else {
      AFL_CUDA(ensure_dyn_smem(trimmed_mean_large_kernel<false>, static_cast<int>(kLargeMaxRows) * 16, smem_attr_done));
      trimmed_mean_large_kernel<false><<<grid, 256, smem, stream>>>(P, dtype == AFL_BF16 ? 1 : 0);
    }
    AFL_LAUNCH_CHECK("trimmed_mean_large_kernel");
    return AFL_OK;
  }
  // S = slots per lane, a multiple of 4 with 32 * S >= n_rows: the work per column is proportional to S, not to n_rows
  // (Bulyan's second stage at N = 1000, f = 240 selects 520 rows: S = 20 instead of 32)
  if (n_rows <= 128) return launch<4>(P, dtype, batch, stream);
  if (n_rows <= 256) return launch<8>(P, dtype, batch, stream);
  if (n_rows <= 384) return launch<12>(P, dtype, batch, stream);
  if (n_rows <= 512) return launch<16>(P, dtype, batch, stream);
  if (n_rows <= 640) return launch<20>(P, dtype, batch, stream);
  if (n_rows <= 768) return launch<24>(P, dtype, batch, stream);
  if (n_rows <= 896) return launch<28>(P, dtype, batch, stream);
  return launch<32>(P, dtype, batch, stream);
}

// A batch with a table whose problems have up to 1024 participating rows each (each[b].tm.n_rows): problem b runs the
// instance that its own row count selects, so its result is its single call's bit for bit.  perm (device, `batch`
// entries) lists the problems class by class, counts[c] (host, kSlotClasses entries) how many have class c; one launch
// per class present, over its problems only.
int trimmed_mean_classes(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, float* out,
                         int batch, int64_t g_batch, int ri_batch, int64_t out_batch, cudaStream_t stream,
                         const ProblemParams* each, const int* perm, const int* counts) {
  if (!G || !out || !each || !perm || !counts || n < 1 || d < 1 || ld < d || batch < 1) {
    set_error("afl_trimmed_mean: bad argument");
    return AFL_ERR_BAD_ARG;
  }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_trimmed_mean: dtype"); return AFL_ERR_UNSUPPORTED; }
  Params P{};
  P.G = G; P.row_index = row_index; P.out = out; P.d = d; P.ld = ld; P.n_total = n;
  P.each = each; P.g_batch = g_batch; P.out_batch = out_batch; P.ri_batch = ri_batch;
  const int64_t es = dtype == AFL_F32 ? 4 : 2;
  P.vec_ok = (reinterpret_cast<uintptr_t>(G) % 16 == 0) && ((ld * es) % 16 == 0) && (batch == 1 || (g_batch * es) % 16 == 0);
  int first = 0;
  for (int c = 0; c < kSlotClasses; first += counts[c], ++c) {
    if (counts[c] < 1) continue;
    const int* pc = perm + first;
    int rc = AFL_OK;
    switch (c) {
      case 0: rc = launch<4>(P, dtype, counts[c], stream, pc); break;
      case 1: rc = launch<8>(P, dtype, counts[c], stream, pc); break;
      case 2: rc = launch<12>(P, dtype, counts[c], stream, pc); break;
      case 3: rc = launch<16>(P, dtype, counts[c], stream, pc); break;
      case 4: rc = launch<20>(P, dtype, counts[c], stream, pc); break;
      case 5: rc = launch<24>(P, dtype, counts[c], stream, pc); break;
      case 6: rc = launch<28>(P, dtype, counts[c], stream, pc); break;
      default: rc = launch<32>(P, dtype, counts[c], stream, pc); break;
    }
    if (rc) return rc;
  }
  return AFL_OK;
}

// trimmed_mean_classes with the class sizes in device memory: perm as there, start[kSlotClasses + 1] (device) the offset
// of each class in perm.  One device-count launch per class, all kSlotClasses of them whether a class is present or
// not, so the host reads nothing and the launches can be captured into a CUDA graph.
int trimmed_mean_classes_dev(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, float* out,
                             int batch, int64_t g_batch, int ri_batch, int64_t out_batch, cudaStream_t stream,
                             const ProblemParams* each, const int* perm, const int* start) {
  if (!G || !out || !each || !perm || !start || n < 1 || d < 1 || ld < d || batch < 1) {
    set_error("afl_trimmed_mean: bad argument");
    return AFL_ERR_BAD_ARG;
  }
  if (dtype != AFL_F32 && dtype != AFL_BF16 && dtype != AFL_F16) { set_error("afl_trimmed_mean: dtype"); return AFL_ERR_UNSUPPORTED; }
  Params P{};
  P.G = G; P.row_index = row_index; P.out = out; P.d = d; P.ld = ld; P.n_total = n;
  P.each = each; P.g_batch = g_batch; P.out_batch = out_batch; P.ri_batch = ri_batch;
  const int64_t es = dtype == AFL_F32 ? 4 : 2;
  P.vec_ok = (reinterpret_cast<uintptr_t>(G) % 16 == 0) && ((ld * es) % 16 == 0) && (batch == 1 || (g_batch * es) % 16 == 0);
  int rc = AFL_OK;
  if ((rc = launch_dev<4>(P, dtype, batch, stream, perm, start, 0))) return rc;
  if ((rc = launch_dev<8>(P, dtype, batch, stream, perm, start, 1))) return rc;
  if ((rc = launch_dev<12>(P, dtype, batch, stream, perm, start, 2))) return rc;
  if ((rc = launch_dev<16>(P, dtype, batch, stream, perm, start, 3))) return rc;
  if ((rc = launch_dev<20>(P, dtype, batch, stream, perm, start, 4))) return rc;
  if ((rc = launch_dev<24>(P, dtype, batch, stream, perm, start, 5))) return rc;
  if ((rc = launch_dev<28>(P, dtype, batch, stream, perm, start, 6))) return rc;
  return launch_dev<32>(P, dtype, batch, stream, perm, start, 7);
}

int trimmed_mean(const void* G, int n, int64_t d, int64_t ld, int dtype, const int* row_index, int n_rows,
                 int corrupted_count, float* out, cudaStream_t stream) {
  return trimmed_mean_batched(G, n, d, ld, dtype, row_index, n_rows, corrupted_count, out, 1, 0, 0, 0, stream, nullptr);
}

}  // namespace tmean
}  // namespace afl
