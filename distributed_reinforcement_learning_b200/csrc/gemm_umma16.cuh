// gemm_umma16.cuh -- gather-GEMM on the Hopper tensor cores with 16-BIT SPLIT operands (wgmma.mma_async f16 / bf16,
// fp32 accumulation in registers): fp32-grade results from half-width operand tiles.
//
//     x = hi + lo + e,   hi = rn16(x),  lo = rn16(x - hi)          (x - hi is exact in fp32)
//     A*B ~= A_lo*B_hi + A_hi*B_lo + A_hi*B_hi                     (dropped: A_lo*B_lo and the e terms)
//
//   format   mantissa   |e|/|x|     dropped A_lo*B_lo    range
//   bf16     8 bits     2^-17       2^-16               fp32's own (no overflow / underflow concerns)
//   fp16     11 bits    2^-22       2^-22               6e-8 .. 65504 (lo underflows gradually below |x| ~ 1e-4:
//                                                       absolute error <= 3e-8; conversion saturates, never inf)
// Both operands of one GEMM use the SAME format (wgmma has one type for A and B); the format is chosen per GEMM.
// Compared with the 3xTF32 core (gemm_umma.cuh): an operand element costs 4 bytes of shared memory (hi + lo) instead
// of 8, so a pipeline stage of the same size covers K = 64 instead of 32, the tensor core reads half the bytes per
// product, each MMA instruction retires K = 16 instead of 8, and 16-bit operands may be MN-major (no transposing
// stores in the producers).
//
// Same structure as gemm_umma_kernel (producer warps 0..PW-1, two consumer warpgroups PW..PW+7 that issue the MMAs and
// run the epilogue, optional bulk-copy loader warp PW+8 for pre-tiled weight images), same loader / epilogue functors.
// Differences:
//   * a stage is filled in two SUB-TILES of K = 32 (so the per-thread register footprint of the gathers stays that of
//     the 3xTF32 kernel); a producer "unit" is 8 consecutive elements of the loader's contiguous dimension = two float4
//     loads -> one 16-byte chunk of hi and one of lo;
//   * K-major tiles : rows of 128 bytes = 64 elements, SWIZZLE_128B (16-byte chunk c of row r at c ^ (r & 7)),
//                     8-row groups 1024 bytes apart; a K = 16 slice j starts at +32 j bytes;
//     MN-major tiles: SWIZZLE_128B atoms of 64 (mn) x 8 (k) = 1024 bytes (k-row kr = 128 contiguous bytes, chunk ^ kr);
//                     atom (g = mn / 64, kg = k / 8) at (kg * (ROWS / 64) + g) * 1024: LBO = 1024, SBO = (ROWS/64)*1024;
//                     a K = 16 slice j covers k-groups 2j, 2j+1 and starts at 2 j SBO   (cute: make_gmma_desc<Major::MN>);
//   * uint8 operands (the frames) are exact in fp16: one plane, two products, 16 bytes -> 16 halves with PRMT + HSUB2;
//   * pre-tiled weight images are always K-major (retile_b16_kernel), whatever the weight's own layout;
//   * an A operand over a 16-bit plane (PlaneA, loaders.cuh: K-major, next to a pre-tiled B) is not gathered at all: the
//     producers cp.async its hi and lo chunks into the stage and arrive on the full barrier when the copies land.
#pragma once
#include "gemm_umma.cuh"
#include "split16.cuh"

namespace drl {
namespace umma16 {

// 4 bytes -> 4 fp16 (exact): PRMT builds 0x64bb = 1024 + b, one HSUB2 per pair removes the 1024
__device__ __forceinline__ uint2 u8x4_to_h4(uint32_t w) {
  uint32_t p0 = __byte_perm(w, 0x64646464u, 0x4140), p1 = __byte_perm(w, 0x64646464u, 0x4342);
  uint32_t r0, r1;
  asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r0) : "r"(p0), "r"(0x64006400u));
  asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r1) : "r"(p1), "r"(0x64006400u));
  return make_uint2(r0, r1);
}

// D (+)= A * B for one warpgroup (M = 64, N, K = 16); F: BF16 / F16, TA / TB: 1 for an MN-major A / B tile
template <int N, class F, int TA, int TB>
__device__ __forceinline__ void mma16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  wg::Wg16<N, F::kBf16, TA, TB>::mma(d, adesc, bdesc, accumulate);
}

// 16 bytes global -> shared without registers; bytes = 0 fills the chunk with zeros
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(umma::smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes)
               : "memory");
}
// one arrival on `bar` once every cp.async this thread issued so far has landed (counts against the barrier's own count)
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(umma::smem_u32(bar)) : "memory");
}

}  // namespace umma16

// An A loader may declare `kPlane` (PlaneA, loaders.cuh): its operand is a 16-bit [hi | lo] plane in global memory, and
// the producers copy its 16-byte chunks into the stages with cp.async instead of gathering fp32 into registers.
template <class L, class = void>
struct loader_plane : std::false_type {};
template <class L>
struct loader_plane<L, std::void_t<decltype(L::kPlane)>> : std::bool_constant<L::kPlane> {};

// One 16-bit operand plane of a stage: ROWS x 64 elements = ROWS x 128 bytes.
template <int ROWS, bool KMAJOR>
struct Umma16Tile {
  static constexpr int BK = 64;
  static constexpr int BYTES = ROWS * 128;
  static constexpr int LBO = KMAJOR ? 16 : 1024;
  static constexpr int SBO = KMAJOR ? 1024 : (ROWS / 64) * 1024;
  static_assert(KMAJOR || ROWS % 64 == 0, "MN-major 16-bit tiles are built from 64-element atoms");
  // byte offset of the 16-byte chunk holding elements [k, k+8) of row `idx` (K-major; k multiple of 8) or elements
  // [idx, idx+8) of k-row `k` (MN-major; idx multiple of 8)
  __device__ static __forceinline__ int chunk_off(int idx, int k) {
    if (KMAJOR) return idx * 128 + ((((k >> 3) ^ idx) & 7) << 4);
    return ((k >> 3) * (ROWS / 64) + (idx >> 6)) * 1024 + (k & 7) * 128 + (((((idx & 63) >> 3) ^ k) & 7) << 4);
  }
  __device__ static __forceinline__ int kslice_off(int j) { return KMAJOR ? j * 32 : j * 2 * SBO; }
};

// TAPSUM: every K tile of 64 starts a fresh accumulator, which is added in fp32 to a running sum in K-tile order once its
// MMAs are complete (two register sets).  For the conv data gradients, whose K tiles are filter taps, this rounds and
// sums exactly as a per-tap GEMM followed by a fixed-order tap sum would.
// PREG (MINB = 2 only): the CTA's registers are split by role with setmaxnreg -- each producer thread keeps PREG, the two
// consumer warpgroups take the rest (CREG each).  0: every thread keeps the count it was launched with.
template <int BN_, int STAGES_, int MINB_ = 1, int PW_ = 4, int LW_ = 0, class AF_ = umma16::BF16, class BF_ = umma16::BF16,
          int PFD_ = 0, bool TAPSUM_ = false, int PREG_ = 0>
struct Umma16Cfg {
  static constexpr int PFD = PFD_;   // register prefetch ring depth in 32-wide K sub-tiles (0: 4 / 3 / 2 by operand kind)
  static constexpr int BM = 128, BN = BN_, BK = 64, SUBK = 32, STAGES = STAGES_, MINB = MINB_;
  static constexpr int PW = PW_, LW = LW_;
  static constexpr bool TAPSUM = TAPSUM_;
  static constexpr int NPROD = PW * 32;
  static constexpr int NT = NPROD + wg::kConsumerThreads + 32 * LW;   // producers + two consumer warpgroups [+ loader]
  static_assert(PW == 4 || PW == 8, "4 or 8 producer warps");
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN must be a power of two in [32,256]");
  // register budgets per thread: at launch (allocated in units of 8), then per role
  static constexpr int PREG = PREG_;
  static constexpr int REGS = 65536 / (NT * MINB);
  static constexpr int CREG = PREG ? ((REGS & ~7) * NT - PREG * NPROD) / wg::kConsumerThreads & ~7 : REGS;
  // setmaxnreg acts on whole warpgroups: the lone loader warp would be a partial one (the producers issue the bulk copy)
  static_assert(PREG == 0 || (MINB == 2 && LW == 0), "per-role registers: two CTAs per SM, no loader warp");
  static_assert(PREG % 8 == 0 && (PREG == 0 || (PREG >= 24 && PREG <= REGS)) && CREG <= 256,
                "setmaxnreg takes multiples of 8 in [24, 256]; the producers give registers away");
  // a consumer needs ~16 registers beside its accumulators; with one count for every role, the producers' state counts too
  static_assert((TAPSUM ? BN : BN / 2) + (PREG ? 16 : 40) <= CREG,
                "accumulator does not fit the consumers' register budget: fewer threads or CTAs");
  // registers of the producers' prefetch ring: with one count for every role it shares the CTA with the accumulators and
  // is capped at ~96; a producer with its own budget keeps ~24 registers for its rows and addresses
  static constexpr int PF_REGS = PREG ? PREG - 24 : 96;
  using AF = AF_;   // 16-bit format of the A operand (uint8 operands are always fp16: exact)
  using BF = BF_;
};

template <class Cfg, class AL, class BL>
struct Umma16Smem {
  using TA = Umma16Tile<Cfg::BM, AL::kContigK>;
  using TB = Umma16Tile<Cfg::BN, loader_pretiled<BL>::value ? true : BL::kContigK>;
  static constexpr bool AEX = loader_exact<AL>::value;
  static constexpr int A_BYTES = TA::BYTES, B_BYTES = TB::BYTES;
  static constexpr int STAGE_BYTES = (AEX ? 1 : 2) * A_BYTES + 2 * B_BYTES;
  static constexpr int AUX_BYTES = 1024 + Cfg::NPROD * 32;   // barriers, column-sum scratch (8 floats / thread)
  static constexpr int EPI_BYTES = 8 * wg::kEpiWarpBytes;    // the dead stages are reused
  static constexpr int BYTES = Cfg::STAGES * STAGE_BYTES + AUX_BYTES + 1024;
  static_assert(Cfg::STAGES * STAGE_BYTES >= EPI_BYTES, "epilogue staging tiles must fit into the pipeline stages");
};

// Optional in-kernel timeline (tools/umma16_timeline.py): when the start-time trace buffer of common.cuh is armed AND
// its word 8001 holds kTrace16Magic, the middle CTA of every launch appends {tag, globaltimer ns} pairs behind word
// 8002: 1 start, 2 set-up done, 600+g gathers of sub-tile g issued, 1000+g sub-tile g: stage free (producer thread 0),
// 2000+g sub-tile g stored, 3000+t MMA warp: stage t full, 4000+t MMAs of stage t issued, 5000+t bulk copy of stage t
// issued, 6000 accumulator complete (epilogue may start), 6001 epilogue done.
constexpr unsigned long long kTrace16Magic = 0xD17A16ull;
struct Trace16 {
  unsigned long long* p;
  __device__ __forceinline__ void operator()(unsigned long long tag) const {
    if (p == nullptr) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(p, 1ULL);
    if (i < 12000ULL) { p[1 + 2 * i] = tag; p[2 + 2 * i] = t; }
  }
};
__device__ __forceinline__ Trace16 trace16_arm() {
  unsigned long long* tr = g_trace_tu;
  Trace16 t{nullptr};
  if (tr != nullptr && tr[8001] == kTrace16Magic && blockIdx.x == gridDim.x / 2 && blockIdx.y == gridDim.y / 2 &&
      blockIdx.z == gridDim.z / 2)
    t.p = tr + 8002;
  return t;
}

template <class Cfg, class AL, class BL, class EP>
__global__ void __launch_bounds__(Cfg::NT, Cfg::MINB)
gemm_umma16_kernel(const AL al, const BL bl, const EP ep, int M, int N, int K, int kchunk, int kstep) {
  kernel_prologue();
  const Trace16 TR = trace16_arm();
  if (threadIdx.x == 0) TR((1ull << 40) | ((unsigned long long)gridDim.x << 20) | (gridDim.y * gridDim.z * 1024 + Cfg::BN));
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, SUBK = Cfg::SUBK, STAGES = Cfg::STAGES, NPROD = Cfg::NPROD;
  constexpr bool AK = AL::kContigK;
  constexpr bool BPT = loader_pretiled<BL>::value;
  constexpr bool BKc = BPT ? true : BL::kContigK;            // layout of the B tile in shared memory
  using SM = Umma16Smem<Cfg, AL, BL>;
  using TA = typename SM::TA;
  using TB = typename SM::TB;
  using AF = typename std::conditional<SM::AEX, umma16::F16, typename Cfg::AF>::type;
  using BF = typename Cfg::BF;
  static_assert(AF::kFormat == BF::kFormat, "kind::f16 traps on mixed f16 x bf16 operands: one format per GEMM");
  constexpr bool AEX = SM::AEX;
  constexpr bool A16 = loader_vec16<AL>::value;              // uint8 operand fetched 16 elements per 128-bit load
  static_assert(!AEX || A16, "exact (uint8) operands use the 16-wide raw loads");
  constexpr bool LWB = BPT && Cfg::LW;
  constexpr bool APL = loader_plane<AL>::value;              // A copied from a 16-bit plane (cp.async)
  static_assert(!APL || (BPT && !EP::kColSum), "a plane A operand pairs with a pre-tiled B");
  // units per sub-tile: 8 elements of the contiguous dimension (16 for the raw uint8 loads)
  constexpr int NUA = BM * SUBK / (A16 ? 16 : 8), NUB = BN * SUBK / 8;
  constexpr int UA = NUA / NPROD, UB = BPT ? 1 : NUB / NPROD;
  static_assert(NUA % NPROD == 0 && (BPT || NUB % NPROD == 0), "units must divide among the producer threads");
  constexpr bool kColSum = EP::kColSum && !BKc && !BPT;
  constexpr int OFF_ALO = SM::A_BYTES, OFF_BHI = (AEX ? 1 : 2) * SM::A_BYTES, OFF_BLO = OFF_BHI + SM::B_BYTES;
  using ARaw = typename std::conditional<A16, uint4, float4>::type;
  constexpr int AR = A16 ? 1 : 2;                             // raw registers (float4 / uint4) per A unit

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* aux = smem + STAGES * SM::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty = full + STAGES;
  float4* cs_scratch = reinterpret_cast<float4*>(aux + 1024);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int z = blockIdx.z;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int k0 = z * kstep;
  const int k1 = min(K, k0 + kchunk);
  const int ntiles = (k1 - k0 + BK - 1) / BK;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      umma::mbar_init(&full[s], NPROD + (LWB ? 1 : 0));
      umma::mbar_init(&empty[s], wg::kConsumerWGs);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) TR(2);

  if (warp < Cfg::PW) {
    // ================= PRODUCERS =================
    if constexpr (Cfg::PREG > 0) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::PREG));
    if constexpr (APL) {
      // A from its plane: unit = (row r, 16-byte chunk c of the stage's K = 64), 8 lanes per row (128 contiguous bytes of
      // hi and of lo for a row's K tile), UP rows per thread.  A stage's chunks are all in flight at once: the prefetch
      // depth is the pipeline's STAGES, and no register holds operand data.
      constexpr int UP = BM * (BK / 8) / NPROD;
      static_assert(BM * (BK / 8) % NPROD == 0, "chunks must divide among the producer threads");
      const int c = tid & 7;
      typename AL::Row prow[UP];
      int poff[UP];
#pragma unroll
      for (int i = 0; i < UP; ++i) {
        const int r = (tid >> 3) + i * (NPROD / 8);
        prow[i] = al.row(z, (m0 + r < M) ? m0 + r : -1);
        poff[i] = TA::chunk_off(r, c * 8);
      }
      const uint16_t* hi = al.plane;
      const uint16_t* lo = al.plane + al.count;
#pragma unroll 1
      for (int t = 0; t < ntiles; ++t) {
        const int s = t % STAGES;
        umma::mbar_wait(&empty[s], ((t / STAGES) & 1) ^ 1);
        if (tid == 0) TR(1000 + 2 * t);
        uint8_t* st = smem + s * SM::STAGE_BYTES;
        if constexpr (!LWB) {
          if (tid == 0) {
            const int kt = (k0 + t * BK) / BK;
            umma::mbar_expect_tx(&full[s], 2 * SM::B_BYTES);
            umma::bulk_g2s(st + OFF_BHI, bl.image + ((size_t)blockIdx.y * bl.ktiles + kt) * (size_t)(2 * SM::B_BYTES),
                           2 * SM::B_BYTES, &full[s]);
          }
        }
        const int k = k0 + t * BK + c * 8;
#pragma unroll
        for (int i = 0; i < UP; ++i) {
          const long long e = (k < k1) ? al.chunk(prow[i], k) : -1ll;
          const uint32_t bytes = e >= 0 ? 16u : 0u;
          const size_t o = e >= 0 ? (size_t)e : 0;
          umma16::cp_async16(st + poff[i], hi + o, bytes);
          umma16::cp_async16(st + OFF_ALO + poff[i], lo + o, bytes);
        }
        umma16::cp_async_arrive_noinc(&full[s]);
        if (tid == 0) TR(2000 + 2 * t + 1);
      }
      asm volatile("cp.async.wait_all;" ::: "memory");
    } else {
      // per-unit state: up to two Row handles (MN-major units span two 4-element loader groups), element offset inside
      // the sub-tile along K, and the byte offset of the unit's 16-byte chunk inside the plane for sub-tile 0
      typename AL::Row arow[UA][AR];
      typename BL::Row brow[UB][2];
      int a_k[UA], a_o[UA], b_k[UB], b_o[UB];
  #pragma unroll
      for (int i = 0; i < UA; ++i) {
        const int u = tid + i * NPROD;
        if constexpr (A16) {
          if (AK) {     // unit = (row, 16-k half of the 32-k sub-tile); lanes = consecutive rows
            const int r = u % BM, half = u / BM;
            arow[i][0] = al.row(z, (m0 + r < M) ? m0 + r : -1);
            a_k[i] = half * 16;
            a_o[i] = r;
          } else {      // unit = (k, 16 consecutive mn)
            const int kk = u % SUBK, q16 = u / SUBK;
            arow[i][0] = al.row(z, (m0 + q16 * 16 < M) ? m0 + q16 * 16 : -1);
            a_k[i] = kk;
            a_o[i] = q16 * 16;
          }
        } else if (AK) {
          // 4 lanes cover one row's 32 k (128 contiguous bytes of fp32); rows are visited in the order 0,4,1,5,2,6,3,7
          // within each group of 8 so that the two rows of a store phase (8 lanes) differ in bit 2 of (row & 7): their
          // chunks then fall into different halves of the 128-byte bank window (conflict-free 16-byte stores)
          const int c4 = u & 3, rs = (u >> 2) & 7, r = (u >> 5) * 8 + ((rs & 1) << 2) + (rs >> 1);
          arow[i][0] = al.row(z, (m0 + r < M) ? m0 + r : -1);
          a_k[i] = c4 * 8;
          a_o[i] = r;
        } else {
          const int q = u % (BM / 8), kk = u / (BM / 8);
          arow[i][0] = al.row(z, (m0 + q * 8 < M) ? m0 + q * 8 : -1);
          arow[i][1] = al.row(z, (m0 + q * 8 + 4 < M) ? m0 + q * 8 + 4 : -1);
          a_k[i] = kk;
          a_o[i] = q * 8;
        }
      }
  #pragma unroll
      for (int i = 0; i < UB; ++i) {
        const int u = tid + i * NPROD;
        if constexpr (BPT) {
          b_k[i] = 0; b_o[i] = 0;
        } else if (BKc) {
          const int c4 = u & 3, rs = (u >> 2) & 7, r = (u >> 5) * 8 + ((rs & 1) << 2) + (rs >> 1);
          brow[i][0] = bl.row(z, (n0 + r < N) ? n0 + r : -1);
          b_k[i] = c4 * 8;
          b_o[i] = r;
        } else {
          const int q = u % (BN / 8), kk = u / (BN / 8);
          brow[i][0] = bl.row(z, (n0 + q * 8 < N) ? n0 + q * 8 : -1);
          brow[i][1] = bl.row(z, (n0 + q * 8 + 4 < N) ? n0 + q * 8 + 4 : -1);
          b_k[i] = kk;
          b_o[i] = q * 8;
        }
      }
      float4 csum[UB][2];
  #pragma unroll
      for (int i = 0; i < UB; ++i) { csum[i][0] = zero4(); csum[i][1] = zero4(); }

      // gather sub-tile g (K range [k0 + 32 g, +32)) into registers
      auto gload = [&](int g, ARaw (&ra)[UA][AR], float4 (&rb)[UB][2]) {
        const int kb = k0 + g * SUBK;
        if (tid == 0) TR(600 + g);
  #pragma unroll
        for (int i = 0; i < UA; ++i) {
          const int k = kb + a_k[i];
          if constexpr (A16) {
            ra[i][0] = (k < k1) ? al.load_raw16(arow[i][0], k) : make_uint4(0u, 0u, 0u, 0u);
          } else if (AK) {
            ra[i][0] = (k < k1) ? al.load(arow[i][0], k) : zero4();
            ra[i][1] = (k + 4 < k1) ? al.load(arow[i][0], k + 4) : zero4();
          } else {
            ra[i][0] = (k < k1) ? al.load(arow[i][0], k) : zero4();
            ra[i][1] = (k < k1) ? al.load(arow[i][1], k) : zero4();
          }
        }
        if constexpr (!BPT) {
  #pragma unroll
          for (int i = 0; i < UB; ++i) {
            const int k = kb + b_k[i];
            if (BKc) {
              rb[i][0] = (k < k1) ? bl.load(brow[i][0], k) : zero4();
              rb[i][1] = (k + 4 < k1) ? bl.load(brow[i][0], k + 4) : zero4();
            } else {
              rb[i][0] = (k < k1) ? bl.load(brow[i][0], k) : zero4();
              rb[i][1] = (k < k1) ? bl.load(brow[i][1], k) : zero4();
            }
          }
        }
      };
      // convert sub-tile g and store it into its stage; the second sub-tile of a stage publishes the stage
      auto publish = [&](int g, const ARaw (&ra)[UA][AR], const float4 (&rb)[UB][2]) {
        const int t = g >> 1, sub = g & 1;
        const int s = t % STAGES;
        uint8_t* st = smem + s * SM::STAGE_BYTES;
        if (sub == 0) {
          umma::mbar_wait(&empty[s], ((t / STAGES) & 1) ^ 1);
          if (tid == 0) TR(1000 + g);
          if constexpr (BPT && !LWB) {
            if (tid == 0) {
              const int kt = (k0 + t * BK) / BK;
              umma::mbar_expect_tx(&full[s], 2 * SM::B_BYTES);
              umma::bulk_g2s(st + OFF_BHI, bl.image + ((size_t)blockIdx.y * bl.ktiles + kt) * (size_t)(2 * SM::B_BYTES),
                             2 * SM::B_BYTES, &full[s]);
            }
          }
        }
        const int ksub = sub * SUBK;   // element offset of this sub-tile inside the stage's K = 64
  #pragma unroll
        for (int i = 0; i < UA; ++i) {
          if constexpr (A16) {
            const uint2 h0 = umma16::u8x4_to_h4(ra[i][0].x), h1 = umma16::u8x4_to_h4(ra[i][0].y);
            const uint2 h2 = umma16::u8x4_to_h4(ra[i][0].z), h3 = umma16::u8x4_to_h4(ra[i][0].w);
            const int o0 = AK ? TA::chunk_off(a_o[i], ksub + a_k[i]) : TA::chunk_off(a_o[i], ksub + a_k[i]);
            const int o1 = AK ? TA::chunk_off(a_o[i], ksub + a_k[i] + 8) : TA::chunk_off(a_o[i] + 8, ksub + a_k[i]);
            *reinterpret_cast<uint4*>(st + o0) = make_uint4(h0.x, h0.y, h1.x, h1.y);
            *reinterpret_cast<uint4*>(st + o1) = make_uint4(h2.x, h2.y, h3.x, h3.y);
          } else {
            uint4 h, l;
            umma16::split8<AF>(ra[i][0], ra[i][1], h, l);
            const int off = TA::chunk_off(a_o[i], ksub + a_k[i]);
            *reinterpret_cast<uint4*>(st + off) = h;
            *reinterpret_cast<uint4*>(st + OFF_ALO + off) = l;
          }
        }
        if constexpr (!BPT) {
  #pragma unroll
          for (int i = 0; i < UB; ++i) {
            uint4 h, l;
            umma16::split8<BF>(rb[i][0], rb[i][1], h, l);
            const int off = TB::chunk_off(b_o[i], ksub + b_k[i]);
            *reinterpret_cast<uint4*>(st + OFF_BHI + off) = h;
            *reinterpret_cast<uint4*>(st + OFF_BLO + off) = l;
            if (kColSum) {
              csum[i][0].x += rb[i][0].x; csum[i][0].y += rb[i][0].y; csum[i][0].z += rb[i][0].z; csum[i][0].w += rb[i][0].w;
              csum[i][1].x += rb[i][1].x; csum[i][1].y += rb[i][1].y; csum[i][1].z += rb[i][1].z; csum[i][1].w += rb[i][1].w;
            }
          }
        }
        if (sub == 1) {
          umma::fence_proxy_async();
          umma::mbar_arrive(&full[s]);
        }
        if (tid == 0) TR(2000 + g);
      };

      // register prefetch ring, in sub-tiles, within Cfg::PF_REGS registers
      constexpr int RPS = 4 * UA * AR + (BPT ? 0 : 8 * UB);      // registers one gathered sub-tile occupies
      constexpr int PF0 = Cfg::PFD > 0 ? Cfg::PFD : (A16 ? 4 : (BPT ? 3 : 2));
      constexpr int PFR = Cfg::PF_REGS;
      constexpr int PF = (PF0 * RPS <= PFR) ? PF0 : (PFR / RPS >= 1 ? PFR / RPS : 1);
      const int nsub = 2 * ntiles;
      ARaw ra[PF][UA][AR];
      float4 rb[PF][UB][2];
  #pragma unroll
      for (int d = 0; d < PF - 1; ++d)
        if (d < nsub) gload(d, ra[d], rb[d]);
  #pragma unroll 1
      for (int g0 = 0; g0 < nsub; g0 += PF) {
  #pragma unroll
        for (int u = 0; u < PF; ++u) {
          const int g = g0 + u;
          if (g < nsub) {
            if (g + PF - 1 < nsub) gload(g + PF - 1, ra[(u + PF - 1) % PF], rb[(u + PF - 1) % PF]);
            publish(g, ra[u], rb[u]);
          }
        }
      }

      // bias-gradient row: column sums of B (dY, exact fp32 values) over this CTA's K range, fixed order
      if (kColSum && blockIdx.x == 0) {
        // a thread's units all have q = tid % (BN / 8) (NPROD is a multiple of BN / 8): 8 columns per thread
        float4 a0 = zero4(), a1 = zero4();
  #pragma unroll
        for (int i = 0; i < UB; ++i) {
          a0.x += csum[i][0].x; a0.y += csum[i][0].y; a0.z += csum[i][0].z; a0.w += csum[i][0].w;
          a1.x += csum[i][1].x; a1.y += csum[i][1].y; a1.z += csum[i][1].z; a1.w += csum[i][1].w;
        }
        cs_scratch[2 * tid] = a0;
        cs_scratch[2 * tid + 1] = a1;
        asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory");
        if (tid < BN / 4) {     // thread handles 4 columns: q = tid / 2, half = tid & 1
          const int q = tid >> 1, half = tid & 1;
          float4 tot = zero4();
          for (int j = q; j < NPROD; j += BN / 8) {
            const float4 v = cs_scratch[2 * j + half];
            tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
          }
          const int n = n0 + q * 8 + half * 4;
          if (n < N) ep.store_colsum(z, n, tot.x);
          if (n + 1 < N) ep.store_colsum(z, n + 1, tot.y);
          if (n + 2 < N) ep.store_colsum(z, n + 2, tot.z);
          if (n + 3 < N) ep.store_colsum(z, n + 3, tot.w);
        }
      }

    }
  } else if (warp >= Cfg::PW + 8) {
    // ================= B LOADER (warp PW+8, Cfg::LW) =================
    if constexpr (LWB) {
      if (lane == 0) {
        for (int t = 0; t < ntiles; ++t) {
          const int s = t % STAGES;
          umma::mbar_wait(&empty[s], ((t / STAGES) & 1) ^ 1);
          const int kt = (k0 + t * BK) / BK;
          TR(5000 + t);
          asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(&full[s])),
                       "r"(2 * SM::B_BYTES) : "memory");
          umma::bulk_g2s(smem + s * SM::STAGE_BYTES + OFF_BHI,
                         bl.image + ((size_t)blockIdx.y * bl.ktiles + kt) * (size_t)(2 * SM::B_BYTES), 2 * SM::B_BYTES,
                         &full[s]);
        }
      }
    }
  } else {
    // ================= CONSUMERS (warps PW .. PW+7: warpgroup cw = rows 64 cw .. 64 cw + 63) =================
    if constexpr (Cfg::PREG > 0) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::CREG));
    const int ct = tid - NPROD, cw = ct >> 7, cwarp = (ct >> 5) & 3;
    // A rows of this warpgroup: K-major +64 rows of 128 bytes; MN-major the second 64-element atom of every k-group
    const uint32_t a_off = AK ? (uint32_t)(cw * 64 * 128) : (uint32_t)(cw * 1024);
    const uint64_t da_base = umma::make_desc(0, TA::LBO, TA::SBO), db_base = umma::make_desc(0, TB::LBO, TB::SBO);
    float acc[BN / 2];
    float tsum[Cfg::TAPSUM ? BN / 2 : 1];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (Cfg::TAPSUM ? BN / 2 : 1); ++i) tsum[i] = 0.f;
    for (int t = 0; t < ntiles; ++t) {
      const int s = t % STAGES;
      umma::mbar_wait(&full[s], (t / STAGES) & 1);
      if constexpr (APL) umma::fence_proxy_async();   // the plane chunks were written by cp.async (generic proxy)
      if (ct == 0) TR(3000 + t);
      const uint32_t st = umma::smem_u32(smem + s * SM::STAGE_BYTES);
      const uint64_t a_hi = umma::desc_at(da_base, st + a_off), a_lo = umma::desc_at(da_base, st + OFF_ALO + a_off);
      const uint64_t b_hi = umma::desc_at(db_base, st + OFF_BHI), b_lo = umma::desc_at(db_base, st + OFF_BLO);
      constexpr int TAm = AK ? 0 : 1, TBm = BKc ? 0 : 1;
      wg::fence_operand(acc);
      wg::fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint64_t ao = (uint64_t)(TA::kslice_off(j) >> 4), bo = (uint64_t)(TB::kslice_off(j) >> 4);
        const uint32_t first = ((t > 0 && !Cfg::TAPSUM) || j > 0) ? 1u : 0u;
        if (!AEX) {                                                    // small terms first
          umma16::mma16<BN, AF, TAm, TBm>(acc, a_lo + ao, b_hi + bo, first);
          umma16::mma16<BN, AF, TAm, TBm>(acc, a_hi + ao, b_lo + bo, 1u);
        } else {
          umma16::mma16<BN, AF, TAm, TBm>(acc, a_hi + ao, b_lo + bo, first);
        }
        umma16::mma16<BN, AF, TAm, TBm>(acc, a_hi + ao, b_hi + bo, 1u);
      }
      wg::commit();
      if constexpr (Cfg::TAPSUM) {
        wg::wait<0>();                                 // this tile's partial sum is complete: add it, hand the stage back
        wg::fence_operand(acc);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) tsum[i] += acc[i];
        if ((ct & 127) == 0) umma::mbar_arrive(&empty[s]);
      } else {
        wg::wait<1>();                                 // the MMAs of stage t-1 are complete: hand it back
        wg::fence_operand(acc);
        if (t > 0 && (ct & 127) == 0) umma::mbar_arrive(&empty[(t - 1) % STAGES]);
      }
      if (ct == 0) TR(4000 + t);
    }
    wg::wait<0>();
    wg::fence_operand(acc);
    // ================= EPILOGUE =================
    wg::consumer_sync();                               // both warpgroups are done with the stages: reuse them
    if (ct == 0) TR(6000);
    uint8_t* stg = smem + (ct >> 5) * wg::kEpiWarpBytes;
    if constexpr (Cfg::TAPSUM) wg_epilogue<BN>(ep, tsum, stg, lane, z, m0 + cw * 64 + cwarp * 16, n0, M, N);
    else wg_epilogue<BN>(ep, acc, stg, lane, z, m0 + cw * 64 + cwarp * 16, n0, M, N);
    if (ct == 0) TR(6001);
  }
}

// ---- pre-tiled weight images, 16-bit: per (n-tile, k64-tile) the K-major [B_hi | B_lo] bytes of a stage ----------------
// element (n, k) of a B operand through its loader, whatever its major
template <class BL>
__device__ __forceinline__ float b_elem(const BL& bl, int n, int k) {
  if (BL::kContigK) {
    const typename BL::Row row = bl.row(0, n);
    const float4 v = bl.load(row, k & ~3);
    const float a[4] = {v.x, v.y, v.z, v.w};
    return a[k & 3];
  }
  const typename BL::Row row = bl.row(0, n & ~3);
  const float4 v = bl.load(row, k);
  const float a[4] = {v.x, v.y, v.z, v.w};
  return a[n & 3];
}
template <int BN, class F, class BL>
__global__ void __launch_bounds__(256) retile_b16_kernel(const BL bl, int N, int K, int ktiles, int ntn,
                                                          uint8_t* __restrict__ image) {
  kernel_prologue();
  using TB = Umma16Tile<BN, true>;
  constexpr int UPT = BN * 8;                        // 8-element units per tile (BN rows x 64 elements)
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)ntn * ktiles * UPT) return;
  const int tile = (int)(g / UPT), lu = (int)(g % UPT);
  const int nt = tile / ktiles, kt = tile - nt * ktiles;
  int r, c;
  if (BL::kContigK) { r = lu >> 3; c = lu & 7; }     // 8 lanes read 64 contiguous k of one row
  else { r = lu % BN; c = lu / BN; }                 // lanes read consecutive n of one k (coalesced for N-contiguous weights)
  const int n = nt * BN + r, kb = kt * 64 + c * 8;
  float x[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = (n < N && kb + i < K) ? b_elem(bl, n, kb + i) : 0.f;
  uint4 h, l;
  umma16::split8<F>(make_float4(x[0], x[1], x[2], x[3]), make_float4(x[4], x[5], x[6], x[7]), h, l);
  uint8_t* dst = image + (size_t)tile * (2 * TB::BYTES);
  const int off = TB::chunk_off(r, c * 8);
  *reinterpret_cast<uint4*>(dst + off) = h;
  *reinterpret_cast<uint4*>(dst + TB::BYTES + off) = l;
}

// The same image from an operand whose ROW index is the contiguous one in memory (kContigK == false: x^T, dz^T, [k][n]
// weights): a thread owns 4 consecutive rows x 8 consecutive k -- eight 128-bit loads (lanes = consecutive row groups of one k:
// coalesced), every loaded value used, four hi + four lo 16-byte chunks stored.  retile_b16_kernel spends one thread per
// (row, 8 k) and uses one element of each float4 it loads.
template <int BN, class F, class BL>
__global__ void __launch_bounds__(256) retile_t16_kernel(const BL bl, int N, int K, int ktiles, int ntn,
                                                          uint8_t* __restrict__ image) {
  static_assert(!BL::kContigK, "transposing variant: the loader's row index is contiguous in memory");
  kernel_prologue();
  using TB = Umma16Tile<BN, true>;
  constexpr int UPT = (BN / 4) * 8;                  // (4-row group, 8-k group) units per tile
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)ntn * ktiles * UPT) return;
  const int tile = (int)(g / UPT), lu = (int)(g % UPT);
  const int nt = tile / ktiles, kt = tile - nt * ktiles;
  const int rq = lu % (BN / 4), c = lu / (BN / 4);
  const int n = nt * BN + rq * 4, kb = kt * 64 + c * 8;
  float x[8][4];
  const typename BL::Row row = bl.row(0, n < N ? n : -1);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = (n < N && kb + i < K) ? bl.load(row, kb + i) : zero4();
    x[i][0] = v.x; x[i][1] = v.y; x[i][2] = v.z; x[i][3] = v.w;
  }
  uint8_t* dst = image + (size_t)tile * (2 * TB::BYTES);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint4 h, l;
    umma16::split8<F>(make_float4(x[0][j], x[1][j], x[2][j], x[3][j]), make_float4(x[4][j], x[5][j], x[6][j], x[7][j]), h, l);
    if (n + j >= N) { h = make_uint4(0u, 0u, 0u, 0u); l = h; }
    const int off = TB::chunk_off(rq * 4 + j, c * 8);
    *reinterpret_cast<uint4*>(dst + off) = h;
    *reinterpret_cast<uint4*>(dst + TB::BYTES + off) = l;
  }
}

template <int BN, class F, class BL>
inline int launch_retile_t16(cudaStream_t s, const BL& bl, int N, int K, uint8_t* image) {
  const int ntn = cdiv(N, BN), ktiles = cdiv(K, 64);
  const long long units = (long long)ntn * ktiles * (BN / 4) * 8;
  DRL_CUDA_CHECK((launch_k(retile_t16_kernel<BN, F, BL>, (unsigned)cdiv64(units, 256), 256, 0, s, bl, N, K, ktiles, ntn, image)));
  return DRL_OK;
}

template <int BN>
inline size_t weight_image16_bytes(int N, int K) {
  return (size_t)cdiv(N, BN) * cdiv(K, 64) * 2 * BN * 128;
}

template <int BN, class F, class BL>
inline int launch_retile_b16(cudaStream_t s, const BL& bl, int N, int K, uint8_t* image) {
  const int ntn = cdiv(N, BN), ktiles = cdiv(K, 64);
  const long long units = (long long)ntn * ktiles * BN * 8;
  // 128-thread blocks: the images of a step are written beside the persistent conv1 kernel, whose 448 x 128 registers leave
  // room for 128 threads x 64 registers per SM but not for a 256-thread block (the second image kernel used to wait ~20 us)
  DRL_CUDA_CHECK((launch_k(retile_b16_kernel<BN, F, BL>, (unsigned)cdiv64(units, 128), 128, 0, s, bl, N, K, ktiles, ntn, image)));
  return DRL_OK;
}

template <class Cfg, class AL, class BL, class EP>
inline int launch_gemm_umma16(cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                              int zcount, int kchunk, int kstep) {
  using SM = Umma16Smem<Cfg, AL, BL>;
  static bool attr_done = false;
  auto kern = gemm_umma16_kernel<Cfg, AL, BL, EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::BYTES));
    attr_done = true;
  }
  constexpr bool bk = loader_pretiled<BL>::value ? false : BL::kContigK;
  if ((AL::kContigK || bk) && (K % 8 != 0 || kchunk % 8 != 0)) {
    set_error("gemm_umma16: K (%d) and kchunk (%d) must be multiples of 8 for K-contiguous operands", K, kchunk);
    return DRL_ERR_INVALID;
  }
  if (loader_pretiled<BL>::value && (kstep % 64 != 0)) {
    set_error("gemm_umma16: split-K step (%d) must be a multiple of 64 with a pre-tiled B", kstep);
    return DRL_ERR_INVALID;
  }
  if (kchunk < 1 || K < 1) { set_error("gemm_umma16: empty K range"); return DRL_ERR_INVALID; }
  // consumers hand a stage back only after the MMAs of the NEXT stage are issued: one stage holds one K tile at most
  if (Cfg::STAGES < 2 && (kchunk > Cfg::BK || (zcount == 1 && K > Cfg::BK))) {
    set_error("gemm_umma16: a single-stage configuration takes K <= %d per split (kchunk %d, K %d)", Cfg::BK, kchunk, K);
    return DRL_ERR_INVALID;
  }
  dim3 grid(cdiv(M, Cfg::BM), cdiv(N, Cfg::BN), zcount);
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT, SM::BYTES, s, al, bl, ep, M, N, K, kchunk, kstep)));
  return DRL_OK;
}

}  // namespace drl
