// Tensor-core Gram kernel (reference: defences.py:16-21 `_krum_create_distances`, the dominant cost of Krum and
// Bulyan): S = G G^T on Hopper warpgroup MMAs (wgmma), lower-triangular 128 x 128 tile pairs, K split over CTAs.
//
//   * The N x N table is cut into T = ceil(N/128) row tiles; only the T(T+1)/2 pairs (I >= J) are computed.
//     CTA = (pair, K split); split s owns the k-blocks s, s+S, s+2S, ... and writes its partial S tile to a private
//     slot, which pair_reduce_kernel sums in a fixed order in float64 (bit-reproducible).  A batch of same-shape
//     problems adds grid dimension y = problem (a 3-D tensor map {d, n, batch}), with one private slot per (problem,
//     pair, split); with more than one tile each problem's bf16x2 centre is its own row of a [batch][d_pad] buffer.
//   * One TMA box {k-block columns x 128 rows} per tile and k-block lands in a 7-slot ring of 32 KB slots (rows past
//     N and columns past D are zero-filled).  Three operand formats (`kMode`):
//       kModeBf16x2  fp32 clients, 64-column k-blocks.  A converter warp rewrites the slot IN PLACE: every 8-row
//                    unit (2 KB of fp32) becomes one SWIZZLE_128B core-matrix atom of b1 (1 KB) followed by one of
//                    b2 (1 KB), with g - c = b1 + b2 + r, |r| <= 2^-17 |g - c| (both roundings to nearest), c = the
//                    mean of the LAST 8 clients' rows (translation invariance of the distances: the cancellation
//                    error of d2 = s_ii + s_jj - 2 s_ij then scales with the distances to an honest client -
//                    main.py:28 makes ids >= f honest - instead of with ||g||^2).  Per 16 columns:
//                        S += b1_I b1_J^T,  S += b1_I b2_J^T,  S += b2_I b1_J^T      (dropped: b2 b2^T, ~2^-17)
//                    With one tile (N <= 128) every pair is on the diagonal tile, so the converters write 2 b2 (exact)
//                    and two products suffice: M += b1 b1^T + b1 (2 b2)^T, and S = (M + M^T) / 2, formed in float64
//                    from the split sums (pair_reduce_kernel keeps both triangles, pair_to_sqdist_kernel adds them).
//                    Its boxes have N rounded up to 8 rows (kSymN); rows past them stay zero from the kernel's start,
//                    and its MMAs are m64nNk16 with N = kSymN, so no tensor work is spent on columns past the box.
//       kModeTf32x2  fp32 clients, 32-column k-blocks delivered by TMA already swizzled (SWIZZLE_128B).  The
//                    converter truncates the box in place to hi = the top 10 mantissa bits and writes lo = g - hi
//                    at the same offsets 16 KB further; per 8 columns S += hi hi^T + hi lo^T + lo hi^T (dropped:
//                    lo lo^T, <= 2^-20 relative).  No centring.
//       kModeBf16In  bf16 clients: TMA delivers ready-made SWIZZLE_128B operand tiles, S += g_I g_J^T exactly
//                    (only the fp32 accumulation rounds), no converter pass.
//       kModeF16In   fp16 clients: the same with FLOAT16 tiles and wgmma .f16 operands (an fp16 product is exact in
//                    fp32 too).
//     With more than one tile EVERY pair - diagonal ones too - issues the same sequence on the same K partition, so two
//     clients with identical rows get bit-identical s_ii, s_jj and s_ij wherever their tiles are, and their distance is
//     exactly 0 (ALIE makes rows 0..f-1 one array; Krum's [1, 0, 2, ...] tie-break depends on it).  Their distances to
//     a third client j are identical unless j lies between them: the higher row of a pair is the I operand, so the two
//     cross products of (j, i) and (k, j), i < j < k, are added in opposite orders (DESIGN 2.1).  The one-tile
//     symmetric form keeps this: identical rows i, k give M_ik = M_ki = M_ii = M_kk bit for bit, and M_ij + M_ji =
//     M_kj + M_jk.  (Across tiles an off-diagonal pair would need all three products to match the diagonal ones.)
//   * Two consumer warpgroups own rows 0..63 and 64..127 of the I tile and issue wgmma.m64n128 with both operands
//     read from shared memory.  The tensor core truncates while it accumulates, so its chains stay short: the
//     register accumulator restarts every `flush` k-blocks and is added (round to nearest) to a running fp32 sum.
//
// Warp roles (384 threads): warp 0 TMA producer, warps 1-3 converters (warp w owns boxes w-1, w+2, ...),
// warpgroups 1 and 2 MMA + accumulation.
// bounded waits trap after 2^35 cycles (~20 s) here: profiler replays with patched SASS run this kernel >100x slower
#define AFL_BAR_TIMEOUT_LOG2 35
#include "afl_common.cuh"

namespace afl {
namespace gram {

constexpr int kPThreads = 384;
constexpr int kConverters = 3;
constexpr int kPSlots = 7;                   // 7 x 32 KB + 1 KB alignment slack fits the 227 KB of an H100 block
constexpr int kPSlotBytes = 128 * 256;       // 128 rows x 64 fp32
constexpr int kPCols = 64;                   // columns per k-block (kModeTf32x2: 32)
constexpr int kPPartElems = 128 * 128;       // S per (pair, split)

struct PairParams {
  int n, tiles, pairs, splits;
  int box_rows;         // rows per TMA box: 128, or with one bf16x2 tile N rounded up to 8
  int kblocks;          // ceil(d / columns per k-block)
  int flush;            // k-blocks per tensor-core accumulation chain
  int center;           // kModeBf16x2: 0 no centring, 1 subtract cvec, 2 (N <= 128) subtract the mean of box rows crow0..
  int crow0;            // first of the last 8 clients' rows (center == 2)
  int single_pass;      // kModeTf32x2: hi hi^T only (plain TF32), for measurement
  const float* cvec;    // centre (mean of the last rows), padded with zeros to a multiple of 64 columns
  float* parts;         // [pairs][splits][128][128]
  const ProblemParams* each;   // kRows: problem b's participating rows are each[b].tm.n_rows
};

__device__ __forceinline__ uint32_t pack_bf16x2_rn_p(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ void sts64_p(uint32_t addr, uint32_t a, uint32_t b) {
  asm volatile("st.shared.v2.b32 [%0], {%1,%2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// wgmma.m64nNk16 (bf16 operands from shared memory, fp32 accumulate) for N = 56, 64, ..., 112: thread t of the
// warpgroup holds N / 2 accumulators.  The asm operand lists are built by macros; IA, IB, IK are the operand numbers
// of the two descriptors and `keep`, which follow the N / 2 accumulators.
#define AFL_R28 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, " \
                "%22, %23, %24, %25, %26, %27"
#define AFL_R32 AFL_R28 ", %28, %29, %30, %31"
#define AFL_R36 AFL_R32 ", %32, %33, %34, %35"
#define AFL_R40 AFL_R36 ", %36, %37, %38, %39"
#define AFL_R44 AFL_R40 ", %40, %41, %42, %43"
#define AFL_R48 AFL_R44 ", %44, %45, %46, %47"
#define AFL_R52 AFL_R48 ", %48, %49, %50, %51"
#define AFL_R56 AFL_R52 ", %52, %53, %54, %55"
#define AFL_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define AFL_C28 AFL_F4(0), AFL_F4(4), AFL_F4(8), AFL_F4(12), AFL_F4(16), AFL_F4(20), AFL_F4(24)
#define AFL_C32 AFL_C28, AFL_F4(28)
#define AFL_C36 AFL_C32, AFL_F4(32)
#define AFL_C40 AFL_C36, AFL_F4(36)
#define AFL_C44 AFL_C40, AFL_F4(40)
#define AFL_C48 AFL_C44, AFL_F4(44)
#define AFL_C52 AFL_C48, AFL_F4(48)
#define AFL_C56 AFL_C52, AFL_F4(52)
#define AFL_WGMMA_BF16_N(N, K, IA, IB, IK)                                                                          \
  __device__ __forceinline__ void wgmma_m64nNk16_bf16(float (&d)[K], uint64_t a_desc, uint64_t b_desc, uint32_t keep) { \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IK ", 0;\n\t"                                               \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" AFL_R##K "}, %" #IA ", %" #IB             \
                 ", p, 1, 1, 0, 0;\n\t}\n"                                                                            \
                 : AFL_C##K : "l"(a_desc), "l"(b_desc), "r"(keep));                                                   \
  }
AFL_WGMMA_BF16_N(56, 28, 28, 29, 30)
AFL_WGMMA_BF16_N(64, 32, 32, 33, 34)
AFL_WGMMA_BF16_N(72, 36, 36, 37, 38)
AFL_WGMMA_BF16_N(80, 40, 40, 41, 42)
AFL_WGMMA_BF16_N(88, 44, 44, 45, 46)
AFL_WGMMA_BF16_N(96, 48, 48, 49, 50)
AFL_WGMMA_BF16_N(104, 52, 52, 53, 54)
AFL_WGMMA_BF16_N(112, 56, 56, 57, 58)
#undef AFL_WGMMA_BF16_N
#undef AFL_F4

// keeps the compiler from touching accumulator registers across a wgmma_wait
template <int K>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[K]) {
#pragma unroll
  for (int i = 0; i < K; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// kSymN > 0: kModeBf16x2 with one tile, the symmetric two-product form on boxes of kSymN = p.box_rows rows (N rounded
// up to 8, 56..112), with wgmma.m64nNk16 for N = kSymN: no tensor work on columns past the box.  (A template
// parameter: a runtime branch between the two MMA sequences makes ptxas fence every k-block's wgmma issue.)
// kRows (a ragged batch, center == 2 only): problem b's centre is the mean of its own last 8 participating rows,
// max(m - 8, 0) .. m - 1 with m = p.each[b].tm.n_rows, instead of rows n - 8 .. n - 1 of the box.
// kRows without kSym (kModeBf16x2 with more than one tile, batch > 1): problem b's centre is row b of the
// [batch][kblocks * 64] cvec buffer that pair_center_kernel wrote (its own last rows, ragged or not).
template <int kMode, int kSymN, bool kRows>
__global__ void __launch_bounds__(kPThreads, 1)
gram_pair_kernel(const __grid_constant__ CUtensorMap tmap, const PairParams p) {
  constexpr bool kSym = kSymN != 0;
  constexpr bool kEachCen = kRows && !kSym;                 // per-problem centre vector
  static_assert(!kSym || (kMode == kModeBf16x2 && kSymN % 8 == 0 && kSymN >= 56 && kSymN <= 112),
                "the symmetric form is a bf16x2 form on 8-row units, and warpgroup 2's rows 64.. must exist");
  constexpr int kAcc = kSym ? kSymN / 2 : 64;               // accumulators per thread (m64nN: N / 2)
  constexpr uint32_t kBoxBytes = kMode == kModeBf16x2 ? kPSlotBytes : kPSlotBytes / 2;
  constexpr int kCols = kMode == kModeTf32x2 ? 32 : kPCols;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t raw_full[kPSlots], conv_done[kPSlots], slot_free[kPSlots];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int pair = blockIdx.x % p.pairs;
  const int split = blockIdx.x / p.pairs;
  int ti = 0;
  while ((ti + 1) * (ti + 2) / 2 <= pair) ++ti;           // pair = ti (ti + 1) / 2 + tj, tj <= ti
  const int tj = pair - ti * (ti + 1) / 2;
  const bool has_b = ti != tj;
  const int nbx = has_b ? 2 : 1;                            // TMA boxes (= ring slots) per k-block
  const int nkb = split < p.kblocks ? (p.kblocks - split + p.splits - 1) / p.splits : 0;
  const int nboxes = nkb * nbx;
  const uint32_t ring = smem_u32(smem);
  // box b of this CTA (b = k-block * nbx + which tile) lives in ring slot b % kPSlots
  auto phase_of = [](int b) -> uint32_t { return static_cast<uint32_t>(b / kPSlots) & 1u; };
  // Converter wait for box b.  The slot's previous box b - kPSlots belongs to another converter warp, and TMA loads do
  // not complete in issue order: while that box is still in flight raw_full is one phase behind, and a parity wait for
  // box b would pass at once.  So first wait until the previous box has been converted (hence has landed).  Parity
  // waits only tell adjacent phases apart; both are valid here: conv_done is at the previous box's phase or one past
  // it (box b, which only this warp converts, has not been), and then raw_full is at box b's phase or one past it.
  auto wait_raw = [&](int b) {
    if (b >= kPSlots) mbar_wait_fast(&conv_done[b % kPSlots], phase_of(b - kPSlots));
    mbar_wait_fast(&raw_full[b % kPSlots], phase_of(b));
  };
  const uint32_t box_bytes = kSym ? static_cast<uint32_t>(p.box_rows) * 256u : kBoxBytes;

  if (kSym) {
    // rows box_rows..127 of every slot: zero bf16 atoms, written once here and never again by TMA or the converters
    for (uint32_t o = box_bytes + threadIdx.x * 16u; o < kPSlotBytes; o += kPThreads * 16u)
      for (int s = 0; s < kPSlots; ++s) sts128(ring + static_cast<uint32_t>(s) * kPSlotBytes + o, make_float4(0.f, 0.f, 0.f, 0.f));
    fence_proxy_async_smem();                               // the wgmma reads them through the async proxy
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < kPSlots; ++s) {
      mbar_init(&raw_full[s], 1);
      mbar_init(&conv_done[s], 32);
      mbar_init(&slot_free[s], 8);                          // lane 0 of each consumer warp
    }
    fence_mbar_init();
  }
  if (warp == 0 && lane == 0) tma_prefetch_desc(&tmap);
  __syncthreads();

  if (wg == 0) {
    if (warp == 0) {
      // ===================== TMA producer: one box per (tile, k-block) =====================
      if (lane == 0) {
        const uint64_t pol = policy_evict_normal();         // every row tile is read by T CTAs: keep it in L2
        for (int b = 0; b < nboxes; ++b) {
          const int s = b % kPSlots;
          mbar_wait(&slot_free[s], phase_of(b) ^ 1u);
          mbar_arrive_expect_tx(&raw_full[s], box_bytes);
          tma_load_3d(smem + static_cast<size_t>(s) * kPSlotBytes, &tmap, &raw_full[s],
                      (split + (b / nbx) * p.splits) * kCols, ((b % nbx) == 0 ? ti : tj) * 128, blockIdx.y, pol);
        }
      }
    } else if (kMode == kModeBf16x2) {
      // ===================== converters: fp32 box -> b1 / b2 atoms, in place =====================
      // A half warp owns one 256-byte fp32 row (16 lanes x 16 bytes); the warp reads 2 rows per LDS.128 and an
      // 8-row unit (2 KB) with 4 of them.  The lane with fp32 chunk c16 owns bf16 bytes [8 c16, 8 c16 + 8) of the
      // 128-byte bf16 row, i.e. half of 16-byte chunk c16/2, which SWIZZLE_128B places at chunk (c16/2)^(row & 7).
      const int w = warp - 1;
      const int rsub = lane >> 4, c16 = lane & 15;
      uint32_t dst_off[4];                                  // destination of row 2u + rsub inside the unit
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t row8 = static_cast<uint32_t>(2 * u + rsub);
        dst_off[u] = row8 * 128u + ((static_cast<uint32_t>(c16 >> 1) ^ row8) << 4) + (static_cast<uint32_t>(c16 & 1) << 3);
      }
      const uint32_t src_lane = static_cast<uint32_t>(rsub) * 256u + static_cast<uint32_t>(c16) * 16u;
      auto load_center = [&](int box) -> float4 {
        if (!(p.center == 1 && box < nboxes)) return make_float4(0.f, 0.f, 0.f, 0.f);
        const int64_t col = static_cast<int64_t>(split + (box / nbx) * p.splits) * kPCols + c16 * 4;
        if constexpr (kEachCen)
          return __ldg(reinterpret_cast<const float4*>(p.cvec + static_cast<int64_t>(blockIdx.y) * p.kblocks * kPCols + col));
        return __ldg(reinterpret_cast<const float4*>(p.cvec + col));
      };
      const int units = box_bytes / 2048u;
      constexpr float two = kSym ? 2.f : 1.f;               // kSym: the second atom is 2 b2 (exact, a power of 2)
      int rows_b = 0, crow0_b = 0;                          // kRows: this problem's row count and first centre row
      if constexpr (kRows && kSym) {
        rows_b = p.each[blockIdx.y].tm.n_rows;
        crow0_b = rows_b > kGramCenterRows ? rows_b - kGramCenterRows : 0;
      }
      float4 cen = load_center(w);
      for (int box = w; box < nboxes; box += kConverters) {
        const int s = box % kPSlots;
        const float4 cnext = load_center(box + kConverters);   // in flight while this box is converted
        wait_raw(box);
        const uint32_t base = ring + static_cast<uint32_t>(s) * kPSlotBytes;
        if (p.center == 2) {
          // one tile: the centre rows are part of this box, so the centre costs no extra HBM traffic; same summation
          // order as gram_center, so the result is the same as pair_center_kernel's
          float4 t[kGramCenterRows];
#pragma unroll
          for (int r = 0; r < kGramCenterRows; ++r)
            t[r] = lds128(base + static_cast<uint32_t>(min((kRows ? crow0_b : p.crow0) + r, (kRows ? rows_b : p.n) - 1)) * 256u +
                          static_cast<uint32_t>(c16) * 16u);
          cen = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int r = 0; r < kGramCenterRows; ++r) { cen.x += t[r].x; cen.y += t[r].y; cen.z += t[r].z; cen.w += t[r].w; }
          const float inv = 1.0f / static_cast<float>(kGramCenterRows);
          cen = gram_center_finite(make_float4(cen.x * inv, cen.y * inv, cen.z * inv, cen.w * inv));
        }
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = lds128(base + src_lane + static_cast<uint32_t>(u) * 512u);
#pragma unroll 1
        for (int unit = 0; unit < units; ++unit) {
          uint32_t h[4][2], l[4][2];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float x0 = v[u].x - cen.x, x1 = v[u].y - cen.y, x2 = v[u].z - cen.z, x3 = v[u].w - cen.w;
            h[u][0] = pack_bf16x2_rn_p(x0, x1);
            h[u][1] = pack_bf16x2_rn_p(x2, x3);
            l[u][0] = pack_bf16x2_rn_p(two * (x0 - __uint_as_float(h[u][0] << 16)), two * (x1 - __uint_as_float(h[u][0] & 0xFFFF0000u)));
            l[u][1] = pack_bf16x2_rn_p(two * (x2 - __uint_as_float(h[u][1] << 16)), two * (x3 - __uint_as_float(h[u][1] & 0xFFFF0000u)));
          }
          const uint32_t ub = base + static_cast<uint32_t>(unit) * 2048u;
          if (unit + 1 < units) {                           // next unit's loads before this unit's stores
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = lds128(ub + 2048u + src_lane + static_cast<uint32_t>(u) * 512u);
          }
          __syncwarp();                                     // every lane has read this unit before anyone overwrites it
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            sts64_p(ub + dst_off[u], h[u][0], h[u][1]);
            sts64_p(ub + 1024u + dst_off[u], l[u][0], l[u][1]);
          }
        }
        cen = cnext;
        fence_proxy_async_smem();
        mbar_arrive(&conv_done[s]);
      }
    } else if (kMode == kModeTf32x2) {
      // ===================== converters: hi = tf32(g) in place, lo = g - hi 16 KB further =====================
      const int w = warp - 1;
      for (int box = w; box < nboxes; box += kConverters) {
        const int s = box % kPSlots;
        wait_raw(box);
        const uint32_t base = ring + static_cast<uint32_t>(s) * kPSlotBytes + static_cast<uint32_t>(lane) * 16u;
#pragma unroll 1
        for (int c0 = 0; c0 < 1024; c0 += 8 * 32) {         // 1024 16-byte chunks per 16 KB box
          float4 v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = lds128(base + (c0 + u * 32) * 16);
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const float4 hi = make_float4(tf32_trunc(v[u].x), tf32_trunc(v[u].y), tf32_trunc(v[u].z), tf32_trunc(v[u].w));
            sts128(base + (c0 + u * 32) * 16, hi);
            sts128(base + kBoxBytes + (c0 + u * 32) * 16, make_float4(v[u].x - hi.x, v[u].y - hi.y, v[u].z - hi.z, v[u].w - hi.w));
          }
        }
        fence_proxy_async_smem();
        mbar_arrive(&conv_done[s]);
      }
    }
  } else {
    // ===================== MMA: warpgroup c owns rows 64c .. 64c+63 of the I tile =====================
    const int c = wg - 1;
    const int wq = warp & 3;
    float acc[kAcc], run[kAcc];
#pragma unroll
    for (int i = 0; i < kAcc; ++i) { acc[i] = 0.f; run[i] = 0.f; }
    // operand layout: kModeBf16x2 alternates 1 KB b1 / b2 atoms (8-row groups 2 KB apart); the other two modes are
    // plain SWIZZLE_128B tiles (8-row groups 1 KB apart), kModeTf32x2 with lo one box further
    constexpr uint32_t kSbo = kMode == kModeBf16x2 ? 2048u : 1024u;
    constexpr uint32_t kSecond = kMode == kModeBf16x2 ? 1024u : kBoxBytes;
    const uint32_t a_off = static_cast<uint32_t>(c) * 8u * kSbo;
    const int ngroups = (nkb + p.flush - 1) / p.flush;
    constexpr bool kDirect = kMode == kModeBf16In || kMode == kModeF16In;     // 16-bit clients: no converter pass
    auto wait_ready = [&](int b) {
      mbar_wait_fast(kDirect ? &raw_full[b % kPSlots] : &conv_done[b % kPSlots], phase_of(b));
    };
    auto release = [&](int it) {
      if (lane == 0) {
        mbar_arrive(&slot_free[(it * nbx) % kPSlots]);
        if (has_b) mbar_arrive(&slot_free[(it * nbx + 1) % kPSlots]);
      }
    };
    for (int g = 0; g < ngroups; ++g) {
      const int it_begin = g * p.flush, it_end = min(it_begin + p.flush, nkb);
      for (int it = it_begin; it < it_end; ++it) {
        wait_ready(it * nbx);
        if (has_b) wait_ready(it * nbx + 1);
        const uint32_t s_i = ring + static_cast<uint32_t>((it * nbx) % kPSlots) * kPSlotBytes;
        const uint32_t s_j = has_b ? ring + static_cast<uint32_t>((it * nbx + 1) % kPSlots) * kPSlotBytes : s_i;
        const uint64_t d_1i = wgmma_desc_sw128(s_i + a_off, kSbo), d_2i = wgmma_desc_sw128(s_i + kSecond + a_off, kSbo);
        const uint64_t d_1j = wgmma_desc_sw128(s_j, kSbo), d_2j = wgmma_desc_sw128(s_j + kSecond, kSbo);
        wgmma_fence();
        const uint32_t first = it != it_begin;            // 0: this chain's first MMA overwrites the accumulator
        if constexpr (kSym) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            wgmma_m64nNk16_bf16(acc, d_1i + 2 * ks, d_1j + 2 * ks, first | ks);    // b1 b1^T
            wgmma_m64nNk16_bf16(acc, d_1i + 2 * ks, d_2j + 2 * ks, 1u);            // b1 (2 b2)^T
          }
        } else if (kMode == kModeTf32x2 && p.single_pass) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks)                    // 4 x 32 bytes = one 128-byte swizzle row of K
            wgmma_m64n128k8_tf32(acc, d_1i + 2 * ks, d_1j + 2 * ks, first | ks);   // hi_I hi_J^T
        } else if (kMode == kModeTf32x2) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            wgmma_m64n128k8_tf32(acc, d_1i + 2 * ks, d_1j + 2 * ks, first | ks);   // hi_I hi_J^T
            wgmma_m64n128k8_tf32(acc, d_1i + 2 * ks, d_2j + 2 * ks, 1u);           // hi_I lo_J^T
            wgmma_m64n128k8_tf32(acc, d_2i + 2 * ks, d_1j + 2 * ks, 1u);           // lo_I hi_J^T
          }
        } else if (kMode == kModeF16In) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks)
            wgmma_m64n128k16_f16(acc, d_1i + 2 * ks, d_1j + 2 * ks, first | ks);     // g_I g_J^T
        } else {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            wgmma_m64n128k16_bf16(acc, d_1i + 2 * ks, d_1j + 2 * ks, first | ks);  // b1_I b1_J^T
            if (kMode == kModeBf16x2) {
              wgmma_m64n128k16_bf16(acc, d_1i + 2 * ks, d_2j + 2 * ks, 1u);        // b1_I b2_J^T
              wgmma_m64n128k16_bf16(acc, d_2i + 2 * ks, d_1j + 2 * ks, 1u);        // b2_I b1_J^T
            }
          }
        }
        wgmma_commit();
        if (it > it_begin) {                                // the previous k-block's operands have been read
          wgmma_wait<1>();
          release(it - 1);
        }
      }
      wgmma_wait<0>();
      release(it_end - 1);
      wgmma_fence_acc(acc);
#pragma unroll
      for (int i = 0; i < kAcc; ++i) run[i] += acc[i];
    }
    // accumulator fragment of m64nN: element i of thread (warp wq, lane) is row 16 wq + lane/4 + 8 ((i/2) % 2),
    // column 8 (i/4) + 2 (lane % 4) + i % 2; kSym writes columns 0..kSymN-1 only
    float* out = p.parts + ((static_cast<size_t>(blockIdx.y) * p.pairs + pair) * p.splits + split) * kPPartElems +
                 static_cast<size_t>(64 * c + 16 * wq + (lane >> 2)) * 128 + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < kAcc; i += 2)
      *reinterpret_cast<float2*>(out + ((i >> 1) & 1) * 8 * 128 + (i >> 2) * 8) = make_float2(run[i], run[i + 1]);
  }
}

// Split reduction of the lower-triangular tile pairs: S[i][j] (i >= j, float64) = sum over splits, in a fixed order
// (threadIdx.y owns a contiguous range, the kPSy partial sums are added in order).  sym (one bf16x2 tile, whose
// partials hold M, not S): every j, so that S[i][j] + S[j][i] = 2 S_ij for pair_to_sqdist_kernel.  blockIdx.z = problem.
constexpr int kPSy = 8;
__global__ void __launch_bounds__(128 * kPSy)
pair_reduce_kernel(const float* __restrict__ parts, int n, int splits, int sym, double* __restrict__ S) {
  __shared__ double sh[kPSy][128];
  const int i = blockIdx.x, tj = blockIdx.y;
  const int ti = i >> 7, ii = i & 127;
  if (tj > ti) return;
  const int jj = threadIdx.x, sy = threadIdx.y;
  const int j = tj * 128 + jj;
  const int pair = (blockIdx.z * gridDim.y * (gridDim.y + 1)) / 2 + ti * (ti + 1) / 2 + tj;
  S += static_cast<size_t>(blockIdx.z) * n * n;
  const float* base = parts + static_cast<size_t>(pair) * splits * kPPartElems + ii * 128 + jj;
  const int s0 = splits * sy / kPSy, s1 = splits * (sy + 1) / kPSy;
  const bool want = (sym || j <= i) && j < n;
  double acc = 0.0;
  if (want)
    for (int s = s0; s < s1; ++s) acc += static_cast<double>(base[static_cast<size_t>(s) * kPPartElems]);
  sh[sy][jj] = acc;
  __syncthreads();
  if (sy == 0 && want) {
    double t = sh[0][jj];
#pragma unroll
    for (int y = 1; y < kPSy; ++y) t += sh[y][jj];
    S[static_cast<size_t>(i) * n + j] = t;
  }
}

// d2_ij = (S_hh + S_ll) - 2 S_hl with h = max(i, j), l = min(i, j): exactly symmetric, zero diagonal, and exactly
// zero between clients whose rows are identical.  sym: 2 S_hl = S[h][l] + S[l][h], the split sums of M_hl and M_lh
// (a floating-point addition is commutative, so identical rows still give bit-identical table rows).
// A row with an inf (its split operands hold inf - inf = NaN) or whose squared norm overflows has a non-finite S_hh:
// its distance to every other client is +inf, as the reference's fp32 norm of a difference that contains an inf.
__global__ void pair_to_sqdist_kernel(const double* __restrict__ S, int n, int sym, double* __restrict__ d2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= n) return;
  S += static_cast<size_t>(blockIdx.z) * n * n;                 // problem blockIdx.z
  d2 += static_cast<size_t>(blockIdx.z) * n * n;
  double v = 0.0;
  if (i != j) {
    const int lo = min(i, j), hi = max(i, j);
    const double s_hh = S[static_cast<size_t>(hi) * n + hi], s_ll = S[static_cast<size_t>(lo) * n + lo];
    const double s_hl = S[static_cast<size_t>(hi) * n + lo];
    v = (isfinite(s_hh) && isfinite(s_ll)) ? (s_hh + s_ll) - (sym ? s_hl + S[static_cast<size_t>(lo) * n + hi] : 2.0 * s_hl)
                                           : __longlong_as_double(0x7ff0000000000000ll);
  }
  d2[static_cast<size_t>(i) * n + j] = v;
}

// centre vectors, grid y = problem: problem b's is the mean of its last min(m, 8) clients, rows max(m - 8, 0) .. m - 1
// of G + b * batch_stride with m = each[b].tm.n_rows (a ragged batch) or n, zero past d (the k-blocks are 64 columns
// wide), at cvec + b * d_pad.  gram_center's arithmetic: problem b's centre is a single call's on its m rows.
__global__ void __launch_bounds__(256)
pair_center_kernel(const float* __restrict__ G, int n, int64_t ld, int64_t batch_stride, int64_t d, int64_t d_pad,
                   const ProblemParams* __restrict__ each, float* __restrict__ cvec) {
  const int64_t col = (static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x) * 4;
  if (col >= d_pad) return;
  const int m = each ? each[blockIdx.y].tm.n_rows : n;
  const int rows = m < kGramCenterRows ? m : kGramCenterRows;
  const float4 c = gram_center(G + blockIdx.y * batch_stride + static_cast<int64_t>(m - rows) * ld, rows, ld, col, d);
  *reinterpret_cast<float4*>(cvec + blockIdx.y * d_pad + col) = c;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// K splits per tile pair: the kernel runs one CTA per SM, so choose the split count whose pairs * splits CTAs fill
// whole waves of SMs best (up to 4 waves; e.g. N = 1000 on 132 SMs: 36 pairs x 11 = 3 full waves instead of 108 CTAs).
// A batch counts pairs x batch CTAs per split, so its partials stay near 4 waves of tiles instead of growing with it.
int pair_splits(int n, int64_t d, int batch) {
  const int tiles = (n + 127) / 128, pairs = tiles * (tiles + 1) / 2 * batch;
  const int64_t kblocks = (d + kPCols - 1) / kPCols;
  const int sms = sm_count();
  int s = 1;
  double best_eff = -1.0;
  for (int w = 1; w <= 4; ++w) {
    int c = sms * w / pairs;
    if (c < 1) c = 1;
    if (c > kblocks) c = static_cast<int>(kblocks);
    const int ctas = pairs * c;
    const double eff = static_cast<double>(ctas) / (static_cast<double>((ctas + sms - 1) / sms) * sms);
    if (eff > best_eff + 1e-9) { best_eff = eff; s = c; }
    if (c == kblocks) break;
  }
  if (const char* e = getenv("AFL_GRAM_SPLITS")) if (atoi(e) > 0) s = atoi(e);
  if (s > kblocks) s = static_cast<int>(kblocks);
  return s < 1 ? 1 : s;
}
// one centre vector per problem (only the multi-tile bf16x2 form of a batch uses more than the first)
size_t pair_center_bytes(int64_t d, int batch) {
  return static_cast<size_t>(batch) * align_up(static_cast<size_t>((d + kPCols - 1) / kPCols * kPCols) * sizeof(float), 256);
}
size_t pair_parts_bytes(int n, int64_t d, int batch) {
  const int tiles = (n + 127) / 128, pairs = tiles * (tiles + 1) / 2;
  return static_cast<size_t>(pairs) * batch * pair_splits(n, d, batch) * kPPartElems * sizeof(float);
}

template <int kMode, int kSymN, bool kRows = false>
static int launch_mode(const CUtensorMap& tmap, const PairParams& p, int batch, cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(kPSlots) * kPSlotBytes + 1024;
  static int smem_attr_done[kMaxDevices] = {0};
  AFL_CUDA(ensure_dyn_smem(gram_pair_kernel<kMode, kSymN, kRows>, static_cast<int>(smem), smem_attr_done));
  {
    ProfScope ps("gram_pair", stream);
    gram_pair_kernel<kMode, kSymN, kRows><<<dim3(p.pairs * p.splits, batch), kPThreads, smem, stream>>>(tmap, p);
  }
  AFL_LAUNCH_CHECK("gram_pair_kernel");
  return AFL_OK;
}

// the one-tile symmetric form: one instance per box height (gram.cu:make_plan runs it for 49 <= N <= 112), and per box
// height one for a ragged batch's per-problem centre
template <bool kRows>
static int launch_sym(const CUtensorMap& tmap, const PairParams& p, int batch, cudaStream_t stream) {
  switch (p.box_rows) {
    case 56: return launch_mode<kModeBf16x2, 56, kRows>(tmap, p, batch, stream);
    case 64: return launch_mode<kModeBf16x2, 64, kRows>(tmap, p, batch, stream);
    case 72: return launch_mode<kModeBf16x2, 72, kRows>(tmap, p, batch, stream);
    case 80: return launch_mode<kModeBf16x2, 80, kRows>(tmap, p, batch, stream);
    case 88: return launch_mode<kModeBf16x2, 88, kRows>(tmap, p, batch, stream);
    case 96: return launch_mode<kModeBf16x2, 96, kRows>(tmap, p, batch, stream);
    case 104: return launch_mode<kModeBf16x2, 104, kRows>(tmap, p, batch, stream);
    case 112: return launch_mode<kModeBf16x2, 112, kRows>(tmap, p, batch, stream);
  }
  set_error("gram_pair_kernel: no one-tile bf16x2 instance for %d clients (49..112)", p.n);
  return AFL_ERR_UNSUPPORTED;
}

// G: `batch` problems of fp32 [n, d] (pitch multiple of 4 elements) or bf16 / fp16 (kModeBf16In / kModeF16In, pitch
// multiple of 8), 16-byte aligned, problem b at G + b * batch_stride elements (batch > 1: a 16-byte multiple >= n * ld).
// parts: pair_parts_bytes(); S and d2_out: batch * n * n doubles; cvec: pair_center_bytes(d, batch) with more than one
// tile, else pair_center_bytes(d, 1).  rows (device, may be NULL): a ragged batch's table, whose tm.n_rows places each
// problem's centre in the bf16x2 forms.  Any other entry S_ij depends on rows i and j only, so the other forms need no
// table.
int launch_pair(const void* Gv, int mode, int batch, int64_t batch_stride, int n, int64_t d, int64_t ld, float* parts,
                double* S, float* cvec, double* d2_out, int flush, int center, int single_pass, cudaStream_t stream,
                const ProblemParams* rows) {
  const float* G = static_cast<const float*>(Gv);
  const bool half16 = mode == kModeBf16In || mode == kModeF16In;    // 16-bit elements
  static EncodeTiledFn enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess) { set_error("cuTensorMapEncodeTiled entry point not found"); return AFL_ERR_CUDA; }
    enc = reinterpret_cast<EncodeTiledFn>(fp);
  }
  const int cols = mode == kModeTf32x2 ? 32 : kPCols;
  PairParams p{};
  p.n = n; p.tiles = (n + 127) / 128; p.pairs = p.tiles * (p.tiles + 1) / 2;
  const int sym = mode == kModeBf16x2 && p.tiles == 1;     // the kernel's kSymN > 0
  p.box_rows = sym ? (n + 7) / 8 * 8 : 128;
  p.splits = pair_splits(n, d, batch);
  p.kblocks = static_cast<int>((d + cols - 1) / cols);
  // `flush` counts 64-column k-blocks of 12 chained bf16 MMAs.  A split-TF32 k-block already chains 12 MMAs over 32 columns,
  // and its truncation bias grows with the chain: one k-block per chain keeps it within that format's 2e-6 budget.
  if (mode == kModeTf32x2) flush = (flush + 3) / 4;
  p.flush = flush < 1 ? 1 : flush;
  p.center = (center && mode == kModeBf16x2) ? (p.tiles == 1 ? 2 : 1) : 0;
  p.crow0 = n > kGramCenterRows ? n - kGramCenterRows : 0;
  p.single_pass = single_pass ? 1 : 0;
  p.parts = parts;
  p.cvec = cvec;
  p.each = rows;
  if (p.center == 1) {
    const int64_t d_pad = (d + kPCols - 1) / kPCols * kPCols;
    pair_center_kernel<<<dim3(static_cast<unsigned>((d_pad / 4 + 255) / 256), batch), 256, 0, stream>>>(
        G, n, ld, batch > 1 ? batch_stride : 0, d, d_pad, rows, cvec);
    AFL_LAUNCH_CHECK("pair_center_kernel");
  }
  CUtensorMap tmap;
  const cuuint64_t es = half16 ? 2 : 4;
  const CUtensorMapDataType elem = mode == kModeBf16In ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                   : mode == kModeF16In ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  const cuuint64_t gdim[3] = {static_cast<cuuint64_t>(d), static_cast<cuuint64_t>(n), static_cast<cuuint64_t>(batch)};
  const cuuint64_t gstride[2] = {static_cast<cuuint64_t>(ld) * es,
                                 static_cast<cuuint64_t>(batch > 1 ? batch_stride : n * ld) * es};
  const cuuint32_t box[3] = {static_cast<cuuint32_t>(cols), static_cast<cuuint32_t>(p.box_rows), 1};
  const cuuint32_t estride[3] = {1, 1, 1};
  CUresult r = enc(&tmap, elem, 3, const_cast<void*>(Gv), gdim,
                   gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   mode == kModeBf16x2 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", static_cast<int>(r)); return AFL_ERR_CUDA; }
  int rc = sym                   ? (rows && p.center == 2 ? launch_sym<true>(tmap, p, batch, stream)
                                                          : launch_sym<false>(tmap, p, batch, stream))
         : mode == kModeBf16x2 ? (batch > 1 ? launch_mode<kModeBf16x2, 0, true>(tmap, p, batch, stream)
                                            : launch_mode<kModeBf16x2, 0>(tmap, p, batch, stream))
         : mode == kModeTf32x2 ? launch_mode<kModeTf32x2, 0>(tmap, p, batch, stream)
         : mode == kModeF16In  ? launch_mode<kModeF16In, 0>(tmap, p, batch, stream)
                               : launch_mode<kModeBf16In, 0>(tmap, p, batch, stream);
  if (rc) return rc;
  pair_reduce_kernel<<<dim3(n, p.tiles, batch), dim3(128, kPSy), 0, stream>>>(parts, n, p.splits, sym, S);
  AFL_LAUNCH_CHECK("pair_reduce_kernel");
  pair_to_sqdist_kernel<<<dim3((n + 127) / 128, n, batch), 128, 0, stream>>>(S, n, sym, d2_out);
  AFL_LAUNCH_CHECK("pair_to_sqdist_kernel");
  return AFL_OK;
}

}  // namespace gram
}  // namespace afl
