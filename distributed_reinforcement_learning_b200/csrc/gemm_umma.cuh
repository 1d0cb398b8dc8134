// gemm_umma.cuh -- gather-GEMM on the Hopper tensor cores (wgmma.mma_async, tf32 operands) with fp32-grade accuracy
// by operand splitting ("3xTF32"):
//
//     x = hi + lo,  hi = rna_tf32(x),  lo = x - hi      (lo is exact in fp32, |lo| <= 2^-11 |x|)
//     A*B ~= A_lo*B_hi + A_hi*B_lo + A_hi*B_hi           (dropped term A_lo*B_lo ~ 2^-22 relative)
//
// all three products accumulate in fp32 in ONE register accumulator.  Same loader / epilogue functor concepts as
// gemm_simt.cuh, so every layer of layers.cu can run on either core.
//
// Structure (one 128 x BN output tile per CTA):
//   warps 0..PW-1 (PW = 4 or 8): PRODUCERS.  Each thread gathers float4 groups of A and B through the loader functors
//               (im2col, concat, transposes, uint8 -> fp32 happen here), splits them into hi/lo and writes both into
//               the stage's shared-memory operand tiles in the canonical K-major SWIZZLE_128B layout (a loader whose
//               contiguous dimension is M or N is transposed on the way: wgmma reads tf32 operands K-major only), then
//               fence.proxy.async and mbarrier-arrive on full[stage].  A weight operand may instead arrive as a
//               pre-split, pre-tiled image with one cp.async.bulk per stage (PretiledB; issued by warp PW+8 when
//               Cfg::LW, else by producer thread 0).
//   warps PW..PW+7: two CONSUMER warpgroups, rows 0-63 and 64-127 of the tile.  Each waits full[stage], issues
//               3 x (BK/8) wgmma.mma_async (M=64, N=BN, K=8) from shared-memory descriptors into its fp32 register
//               accumulator, keeps one stage of MMAs in flight and hands the previous stage back (empty[stage]).
//               After the last K tile it drains the accumulator through a swizzled shared tile (wg_epilogue) into the
//               epilogue functor (bias/ReLU/mask/split-K partial ...).
//
// Canonical SWIZZLE_128B K-major layout (CuTe GMMA::Layout_K_SW128_Atom), BK = 32 floats: row r is 128 contiguous
// bytes (32 floats of K) at r*128; the 16-byte chunk c of row r is stored at chunk position c ^ (r & 7)
// (Swizzle<3,4,3>: address bits [4,7) ^= bits [7,10)).  8-row groups are 1024 bytes apart (SBO = 1024).  A K=8 MMA
// slice j starts at +32*j bytes.  All operand tiles are 1024-byte aligned (base_offset = 0).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "wgmma_ops.cuh"

namespace drl {
namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One lane of a converged warp, chosen by the hardware (elect.sync).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// descriptor = constant part (everything but the start address) + (shared-memory byte address >> 4)
__device__ __forceinline__ uint64_t desc_at(uint64_t base, uint32_t saddr) { return base + (uint64_t)(saddr >> 4); }

// shared-memory matrix descriptor of wgmma (cute::GMMA::GmmaDescriptor): start address, leading / stride byte offsets,
// base_offset 0, layout type 1 = SWIZZLE_128B (bits 62-63)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ float tf32_hi(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ void split4(const float4& x, float4& h, float4& l) {
  h.x = tf32_hi(x.x); h.y = tf32_hi(x.y); h.z = tf32_hi(x.z); h.w = tf32_hi(x.w);
  l.x = x.x - h.x; l.y = x.y - h.y; l.z = x.z - h.z; l.w = x.w - h.w;
}

}  // namespace umma

// ---- warpgroup MMA plumbing shared by every tensor-core kernel ----------------------------------------------------------
namespace wg {
constexpr int kConsumerWGs = 2;                       // two consumer warpgroups: rows 0-63 and 64-127 of a 128-row tile
constexpr int kConsumerThreads = 128 * kConsumerWGs;
constexpr int kEpiWarpBytes = 16 * 128;               // per consumer warp: one 16-row x 32-column staging tile

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// named barrier over the consumer warpgroups only (id 2; id 1 is the producers' column-sum barrier)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 2, %0;" ::"n"(kConsumerThreads) : "memory"); }
}  // namespace wg

// One operand tile of a stage: ROWS (128 for A, BN for B) x 32 floats, K-major SWIZZLE_128B, rows of 128 bytes, 16-byte
// chunks XOR (row & 7).  KMAJOR says how the LOADER delivers the operand: K-major loaders hand over 4 consecutive k of
// one row (one 16-byte chunk); the others hand over 4 consecutive rows of one k, which put() scatters into the four rows
// (tf32 wgmma has no transposed operand mode).
template <int ROWS, bool KMAJOR>
struct UmmaTile {
  static constexpr int BK = 32;
  static constexpr int BYTES = ROWS * BK * 4;
  static constexpr int LBO = 16;                       // unused by the hardware for swizzled K-major tiles
  static constexpr int SBO = 1024;
  // K-major: byte offset of the chunk holding [k, k+4) of row idx (k multiple of 4).  Otherwise: byte offset of element
  // (row idx, k) with idx a multiple of 4 -- put() derives the other three rows from it.
  __device__ static __forceinline__ int chunk_off(int idx, int k) {
    const int c = idx * 128 + ((((k >> 2) ^ idx) & 7) << 4);
    return KMAJOR ? c : c + (k & 3) * 4;
  }
  __device__ static __forceinline__ void put(uint8_t* base, int off, const float4& v) {
    if (KMAJOR) {
      *reinterpret_cast<float4*>(base + off) = v;
    } else {
      // rows idx+j (idx % 4 == 0): chunk c ^ j, same offset inside the chunk
      const int c = (off >> 4) & 7, b = off & ~0x70;
      *reinterpret_cast<float*>(base + b + ((c ^ 0) << 4)) = v.x;
      *reinterpret_cast<float*>(base + b + 128 + ((c ^ 1) << 4)) = v.y;
      *reinterpret_cast<float*>(base + b + 256 + ((c ^ 2) << 4)) = v.z;
      *reinterpret_cast<float*>(base + b + 384 + ((c ^ 3) << 4)) = v.w;
    }
  }
  // descriptor start offset of the j-th K=8 slice
  __device__ static __forceinline__ int kslice_off(int j) { return j * 32; }
};

template <int BN_, int STAGES_, int MINB_ = 1, int PW_ = 4, int LW_ = 0>
struct UmmaCfg {
  static constexpr int BM = 128, BN = BN_, BK = 32, STAGES = STAGES_, MINB = MINB_;
  static constexpr int PW = PW_;            // producer warps (4 or 8), warps 0..PW-1
  static constexpr int LW = LW_;            // 1: warp PW+8 issues the bulk copies of a pre-tiled B (see the kernel)
  static constexpr int NPROD = PW * 32;
  static constexpr int NT = NPROD + wg::kConsumerThreads + 32 * LW;   // + two consumer warpgroups [+ the B loader warp]
  static_assert(PW == 4 || PW == 8, "4 or 8 producer warps");
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN must be a power of two in [32,256]");
  // the BN / 2 accumulator registers of a consumer thread must fit the per-thread register budget of the launch
  static_assert(BN / 2 + 40 <= 65536 / (NT * MINB), "accumulator does not fit the register budget: fewer threads or CTAs");
};

// A loader may declare `static constexpr bool kExactTf32 = true` when its values are exactly representable in
// tf32 (the uint8 frame bytes): then lo == 0, the lo tile is not written and the A_lo*B_hi product is skipped
// ("2xTF32").
template <class L, class = void>
struct loader_exact : std::false_type {};
template <class L>
struct loader_exact<L, std::void_t<decltype(L::kExactTf32)>> : std::bool_constant<L::kExactTf32> {};

// A loader may also declare `kVec16`: it then provides load_raw16()/unpack16() that fetch 16 consecutive
// elements of the contiguous dimension with ONE 128-bit load (the uint8 frames: 4x fewer load instructions).
template <class L, class = void>
struct loader_vec16 : std::false_type {};
template <class L>
struct loader_vec16<L, std::void_t<decltype(L::kVec16)>> : std::bool_constant<L::kVec16> {};

// A B loader may declare `kPretiled`: the operand (a weight matrix) has already been split into hi/lo and stored in
// global memory as per-(n-tile, k-tile) IMAGES of the shared-memory stage layout (retile_b_kernel below, run once
// per parameter update).  The producers then do not touch B at all: one thread fetches [B_hi | B_lo] of a stage
// with a single cp.async.bulk (TMA bulk copy) that completes on the stage's full barrier (complete_tx).
template <class L, class = void>
struct loader_pretiled : std::false_type {};
template <class L>
struct loader_pretiled<L, std::void_t<decltype(L::kPretiled)>> : std::bool_constant<L::kPretiled> {};

template <class Base>
struct PretiledB {
  static constexpr bool kContigK = Base::kContigK;
  static constexpr bool kPretiled = true;
  const uint8_t* image;   // [n-tiles][k-tiles][2 * B_BYTES]
  int ktiles;             // K tiles (of 32) in the image
  struct Row {};
  __device__ __forceinline__ Row row(int, int) const { return Row{}; }
  __device__ __forceinline__ float4 load(const Row&, int) const { return zero4(); }
};

namespace umma {
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// global -> shared bulk copy (TMA engine), completion counted in bytes on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
}  // namespace umma

// An epilogue functor may provide `bias4(z, n)` + `store4b(z, m, n, o, bias)`: the per-column bias of a lane is the same
// for all rows it stores, so it is fetched ONCE per block instead of once per element.
template <class EP, class = void>
struct ep_has_bias4 : std::false_type {};
template <class EP>
struct ep_has_bias4<EP, std::void_t<decltype(std::declval<const EP&>().bias4(0, 0))>> : std::true_type {};

// Second half of an epilogue store: a ROWS x 32 block staged in shared memory (row r = 128 bytes, 16-byte chunks XOR
// (r & 7)) is read back row-wise, 8 lanes per 128-byte row segment, and handed to the functor (coalesced stores).
template <int ROWS, class EP>
__device__ __forceinline__ void epilogue_drain(const EP& ep, const uint8_t* stg, int lane, int z, int row0, int col0,
                                               int M, int N) {
  const int c = lane & 7, rr = lane >> 3;
  const int n = col0 + c * 4;
  float4 bias = zero4();
  if constexpr (ep_has_bias4<EP>::value) {
    if (n + 3 < N) bias = ep.bias4(z, n);
  }
#pragma unroll
  for (int i = 0; i < ROWS / 4; ++i) {
    const int r = i * 4 + rr;
    const float4 o4 = *reinterpret_cast<const float4*>(stg + r * 128 + ((c ^ (r & 7)) << 4));
    const int m = row0 + r;
    if (m < M) {
      const float o[4] = {o4.x, o4.y, o4.z, o4.w};
      if (n + 3 < N) {
        if constexpr (ep_has_bias4<EP>::value) ep.store4b(z, m, n, o, bias);
        else ep.template store<4>(z, m, n, o);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (n + q < N) {
            const float o1[1] = {o[q]};
            ep.template store<1>(z, m, n + q, o1);
          }
      }
    }
  }
}

// Epilogue of one consumer warp: its 16 rows (row0 ..) of a 64 x BN wgmma accumulator (fragment: d[4c + e] holds row
// lane/4 (+8 for e >= 2), column 8c + 2 (lane % 4) + (e & 1)), 32 columns at a time through its 2 KB staging tile.
// FOLD: the accumulator holds [X | Y] of width BN and the epilogue sees X + Y (width BN / 2).
template <int BN, bool FOLD = false, class EP>
__device__ __forceinline__ void wg_epilogue(const EP& ep, const float (&acc)[BN / 2], uint8_t* stg, int lane, int z,
                                            int row0, int n0, int M, int N) {
  constexpr int W = FOLD ? BN / 2 : BN;
  const int r = lane >> 2, q = lane & 3;
  // fully unrolled: a runtime index into acc would put the accumulator in local memory, and ptxas then serialises
  // every wgmma of the main loop (warning C7514), which cost the 16-bit GEMMs about a quarter of their time on H100
#pragma unroll
  for (int cb = 0; cb < W / 32; ++cb) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = (cb * 4 + c) * 4;
      float2 lo = make_float2(acc[i], acc[i + 1]), hi = make_float2(acc[i + 2], acc[i + 3]);
      if constexpr (FOLD) {
        constexpr int H = BN / 4;   // the Y half starts BN / 2 columns = BN / 16 column groups = BN / 4 registers later
        lo.x += acc[i + H]; lo.y += acc[i + H + 1]; hi.x += acc[i + H + 2]; hi.y += acc[i + H + 3];
      }
      const int chunk = 2 * c + (q >> 1), in = (q & 1) * 8;
      *reinterpret_cast<float2*>(stg + r * 128 + ((chunk ^ (r & 7)) << 4) + in) = lo;
      *reinterpret_cast<float2*>(stg + (r + 8) * 128 + ((chunk ^ (r & 7)) << 4) + in) = hi;
    }
    __syncwarp();
    epilogue_drain<16>(ep, stg, lane, z, row0, n0 + cb * 32, M, N);
    __syncwarp();
  }
}

template <class Cfg, class AL, class BL>
struct UmmaSmem {
  using TA = UmmaTile<Cfg::BM, AL::kContigK>;
  using TB = UmmaTile<Cfg::BN, BL::kContigK>;
  static constexpr bool AEX = loader_exact<AL>::value;
  static constexpr int A_BYTES = TA::BYTES, B_BYTES = TB::BYTES;       // multiples of 1024
  static constexpr int STAGE_BYTES = (AEX ? 1 : 2) * A_BYTES + 2 * B_BYTES;   // hi (and lo) copies of the operands
  static constexpr int AUX_BYTES = 1024 + (BL::kContigK ? 0 : Cfg::NPROD * 16);   // barriers, colsum scratch
  static constexpr int BYTES = Cfg::STAGES * STAGE_BYTES + AUX_BYTES + 1024;      // + alignment slack
  static_assert(Cfg::STAGES * STAGE_BYTES >= 8 * wg::kEpiWarpBytes, "epilogue staging tiles live in the dead stages");
};

// The 3xTF32 MMAs of one stage for consumer warpgroup `cw` (A rows 64 cw ..): 3 (2 for an exact A) products per K=8 slice.
template <int BN, bool AEX, int BK, class TA, class TB>
__device__ __forceinline__ void tf32_stage_mmas(float (&acc)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                uint32_t b_lo, bool first_tile) {
  const uint64_t da = umma::make_desc(0, TA::LBO, TA::SBO), db = umma::make_desc(0, TB::LBO, TB::SBO);
#pragma unroll
  for (int j = 0; j < BK / 8; ++j) {
    const uint32_t ao = TA::kslice_off(j), bo = TB::kslice_off(j);
    const uint32_t first = (!first_tile || j > 0) ? 1u : 0u;
    if (!AEX) {                                                    // small terms first
      wg::WgTf32<BN>::mma(acc, umma::desc_at(da, a_lo + ao), umma::desc_at(db, b_hi + bo), first);
      wg::WgTf32<BN>::mma(acc, umma::desc_at(da, a_hi + ao), umma::desc_at(db, b_lo + bo), 1u);
    } else {
      wg::WgTf32<BN>::mma(acc, umma::desc_at(da, a_hi + ao), umma::desc_at(db, b_lo + bo), first);
    }
    wg::WgTf32<BN>::mma(acc, umma::desc_at(da, a_hi + ao), umma::desc_at(db, b_hi + bo), 1u);
  }
}

template <class Cfg, class AL, class BL, class EP>
__global__ void __launch_bounds__(Cfg::NT, Cfg::MINB)
gemm_umma_kernel(const AL al, const BL bl, const EP ep, int M, int N, int K, int kchunk, int kstep) {
  kernel_prologue();
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES, NPROD = Cfg::NPROD;
  constexpr bool AK = AL::kContigK, BKc = BL::kContigK;
  using SM = UmmaSmem<Cfg, AL, BL>;
  using TA = typename SM::TA;
  using TB = typename SM::TB;
  constexpr bool AEX = SM::AEX;
  constexpr int NGA = BM * BK / 4, NGB = BN * BK / 4;       // float4 groups per stage
  constexpr bool A16 = loader_vec16<AL>::value;              // 16-element (one 128-bit load) A groups
  constexpr bool BPT = loader_pretiled<BL>::value;           // B arrives as pre-split stage images via cp.async.bulk
  // with Cfg::LW a dedicated warp (PW+8) issues the bulk copies and arrives on the barrier itself; otherwise producer
  // thread 0 does, in front of its own gathers
  constexpr bool LWB = BPT && Cfg::LW;
  constexpr int GA = (A16 ? NGA / 4 : NGA) / NPROD, GB = BPT ? 1 : NGB / NPROD;   // groups per producer thread
  static_assert((A16 ? NGA / 4 : NGA) % NPROD == 0 && NGB % NPROD == 0, "groups must divide among producers");
  static_assert(!A16 || AEX, "16-wide raw loads are only used for exact (uint8) operands");
  using ARaw = typename std::conditional<A16, uint4, float4>::type;
  constexpr bool kColSum = EP::kColSum && !BKc && !BPT;
  constexpr int OFF_ALO = SM::A_BYTES, OFF_BHI = (AEX ? 1 : 2) * SM::A_BYTES, OFF_BLO = OFF_BHI + SM::B_BYTES;

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

  if (warp < Cfg::PW) {
    // ================= PRODUCERS =================
    // K-major operand : group g -> row g/8, chunk g%8  (8 lanes cover one 128-byte row: coalesced global
    //                   read of 128 contiguous bytes, conflict-free swizzled 16-byte stores)
    // MN-major operand: group g -> k = g/(ROWS/4), quad q = g%(ROWS/4)  (8 lanes cover 32 contiguous mn
    //                   values of one k: coalesced)
    typename AL::Row arow[GA];
    typename BL::Row brow[GB];
    int a_k[GA], a_o[GA], b_k[GB], b_o[GB];
#pragma unroll
    for (int i = 0; i < GA; ++i) {
      const int g = tid + i * NPROD;
      if (A16) {
        if (AK) {   // group = (row, 16-k half): 32 lanes = 32 consecutive rows
          const int r = g % BM, half = g / BM;
          arow[i] = al.row(z, (m0 + r < M) ? m0 + r : -1);
          a_k[i] = half * 16;
          a_o[i] = r;
        } else {    // group = (k, 16 consecutive mn): 32 lanes = the 32 k of the tile for the same 16 mn values
          const int kk = g % BK, q16 = g / BK;
          arow[i] = al.row(z, (m0 + q16 * 16 < M) ? m0 + q16 * 16 : -1);
          a_k[i] = kk;
          a_o[i] = q16 * 16;
        }
      } else if (AK) {
        const int r = g >> 3, kq = g & 7;
        arow[i] = al.row(z, (m0 + r < M) ? m0 + r : -1);
        a_k[i] = kq * 4;
        a_o[i] = TA::chunk_off(r, kq * 4);
      } else {
        const int q = g % (BM / 4), kk = g / (BM / 4);
        arow[i] = al.row(z, (m0 + q * 4 < M) ? m0 + q * 4 : -1);
        a_k[i] = kk;
        a_o[i] = TA::chunk_off(q * 4, kk);
      }
    }
#pragma unroll
    for (int i = 0; i < GB; ++i) {
      const int g = tid + i * NPROD;
      if (BPT) {
        b_k[i] = 0; b_o[i] = 0;
      } else if (BKc) {
        const int r = g >> 3, kq = g & 7;
        brow[i] = bl.row(z, (n0 + r < N) ? n0 + r : -1);
        b_k[i] = kq * 4;
        b_o[i] = TB::chunk_off(r, kq * 4);
      } else {
        const int q = g % (BN / 4), kk = g / (BN / 4);
        brow[i] = bl.row(z, (n0 + q * 4 < N) ? n0 + q * 4 : -1);
        b_k[i] = kk;
        b_o[i] = TB::chunk_off(q * 4, kk);
      }
    }
    float4 csum[GB];
#pragma unroll
    for (int i = 0; i < GB; ++i) csum[i] = zero4();

    // gather tile t into registers
    auto gload = [&](int t, ARaw (&ra)[GA], float4 (&rb)[GB]) {
      const int kb = k0 + t * BK;
#pragma unroll
      for (int i = 0; i < GA; ++i) {
        const int k = kb + a_k[i];
        if constexpr (A16) ra[i] = (k < k1) ? al.load_raw16(arow[i], k) : make_uint4(0u, 0u, 0u, 0u);
        else ra[i] = (k < k1) ? al.load(arow[i], k) : zero4();
      }
      if constexpr (!BPT) {
#pragma unroll
        for (int i = 0; i < GB; ++i) {
          const int k = kb + b_k[i];
          rb[i] = (k < k1) ? bl.load(brow[i], k) : zero4();
        }
      }
    };
    // split tile t into hi/lo and publish it in its shared-memory stage
    auto publish = [&](int t, const ARaw (&ra)[GA], const float4 (&rb)[GB]) {
      const int s = t % STAGES;
      const uint32_t ph = (t / STAGES) & 1;
      umma::mbar_wait(&empty[s], ph ^ 1);
      uint8_t* st = smem + s * SM::STAGE_BYTES;
      if constexpr (BPT && !LWB) {
        if (tid == 0) {   // one bulk copy brings [B_hi | B_lo] of this (n-tile, k-tile); bytes complete on full[s]
          const int kt = (k0 + t * BK) / BK;
          umma::mbar_expect_tx(&full[s], 2 * SM::B_BYTES);
          umma::bulk_g2s(st + OFF_BHI, bl.image + ((size_t)blockIdx.y * bl.ktiles + kt) * (size_t)(2 * SM::B_BYTES),
                         2 * SM::B_BYTES, &full[s]);
        }
      }
#pragma unroll
      for (int i = 0; i < GA; ++i) {
        if constexpr (A16) {
          float4 f[4];
          AL::unpack16(ra[i], f);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int off = AK ? TA::chunk_off(a_o[i], a_k[i] + 4 * j) : TA::chunk_off(a_o[i] + 4 * j, a_k[i]);
            TA::put(st, off, f[j]);
          }
        } else if constexpr (AEX) {
          TA::put(st, a_o[i], ra[i]);
        } else {
          float4 h, l;
          umma::split4(ra[i], h, l);
          TA::put(st, a_o[i], h);
          TA::put(st + OFF_ALO, a_o[i], l);
        }
      }
      if constexpr (!BPT) {
#pragma unroll
        for (int i = 0; i < GB; ++i) {
          float4 h, l;
          umma::split4(rb[i], h, l);
          TB::put(st + OFF_BHI, b_o[i], h);
          TB::put(st + OFF_BLO, b_o[i], l);
          if (kColSum) { csum[i].x += rb[i].x; csum[i].y += rb[i].y; csum[i].z += rb[i].z; csum[i].w += rb[i].w; }
        }
      }
      umma::fence_proxy_async();       // generic-proxy writes -> visible to the tensor-core (async) proxy
      umma::mbar_arrive(&full[s]);
    };

    // register prefetch ring of depth PF: the gathers of tiles t+1 .. t+PF-1 are in flight while tile t is split
    // and stored.  The accumulators live in registers of the same CTA, so the ring is capped at ~96 registers.
    constexpr int RPT = 4 * (GA + (BPT ? 0 : GB));             // registers one gathered tile occupies
    constexpr int PF0 = A16 ? 4 : (BPT ? 3 : 2);
    constexpr int PF = (PF0 * RPT <= 96) ? PF0 : (96 / RPT >= 1 ? 96 / RPT : 1);
    ARaw ra[PF][GA];
    float4 rb[PF][GB];
#pragma unroll
    for (int d = 0; d < PF - 1; ++d)
      if (d < ntiles) gload(d, ra[d], rb[d]);
#pragma unroll 1
    for (int t0 = 0; t0 < ntiles; t0 += PF) {
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int t = t0 + u;
        if (t < ntiles) {
          if (t + PF - 1 < ntiles) gload(t + PF - 1, ra[(u + PF - 1) % PF], rb[(u + PF - 1) % PF]);
          publish(t, ra[u], rb[u]);
        }
      }
    }

    // bias-gradient row: column sums of B (dY) over this CTA's K range, reduced in fixed order
    if (kColSum && blockIdx.x == 0) {
      // thread's groups: q = (tid + i*NPROD) % (BN/4).  NPROD is a multiple of BN/4, so q = tid % (BN/4) for all i.
      float4 acc = zero4();
#pragma unroll
      for (int i = 0; i < GB; ++i) { acc.x += csum[i].x; acc.y += csum[i].y; acc.z += csum[i].z; acc.w += csum[i].w; }
      cs_scratch[tid] = acc;
      asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory");
      if (tid < BN / 4) {
        float4 tot = zero4();
        for (int j = tid; j < NPROD; j += BN / 4) {
          const float4 v = cs_scratch[j];
          tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
        }
        const int n = n0 + tid * 4;
        if (n < N) ep.store_colsum(z, n, tot.x);
        if (n + 1 < N) ep.store_colsum(z, n + 1, tot.y);
        if (n + 2 < N) ep.store_colsum(z, n + 2, tot.z);
        if (n + 3 < N) ep.store_colsum(z, n + 3, tot.w);
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
    const int ct = tid - NPROD, cw = ct >> 7, cwarp = (ct >> 5) & 3;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int t = 0; t < ntiles; ++t) {
      const int s = t % STAGES;
      umma::mbar_wait(&full[s], (t / STAGES) & 1);
      const uint32_t st = umma::smem_u32(smem + s * SM::STAGE_BYTES);
      const uint32_t a_hi = st + cw * 64 * 128;
      wg::fence_operand(acc);
      wg::fence();
      tf32_stage_mmas<BN, AEX, BK, TA, TB>(acc, a_hi, a_hi + OFF_ALO, st + OFF_BHI, st + OFF_BLO, t == 0);
      wg::commit();
      wg::wait<1>();                                   // the MMAs of stage t-1 are complete: hand it back
      wg::fence_operand(acc);
      if (t > 0 && (ct & 127) == 0) umma::mbar_arrive(&empty[(t - 1) % STAGES]);
    }
    wg::wait<0>();
    wg::fence_operand(acc);
    // ================= EPILOGUE =================
    // both warpgroups' MMAs are complete, so the pipeline stages are dead: their first bytes become the staging tiles
    wg::consumer_sync();
    uint8_t* stg = smem + (ct >> 5) * wg::kEpiWarpBytes;
    wg_epilogue<BN>(ep, acc, stg, lane, z, m0 + cw * 64 + cwarp * 16, n0, M, N);
  }
}

// Writes the pre-split, pre-tiled, pre-swizzled image of a B operand: for every (n-tile, k-tile) the exact bytes the
// producers would have put into [B_hi | B_lo] of a stage.  Runs once per parameter update.
template <int BN, class BL>
__global__ void __launch_bounds__(256) retile_b_kernel(const BL bl, int N, int K, int ktiles, int ntn,
                                                        uint8_t* __restrict__ image) {
  kernel_prologue();
  using TB = UmmaTile<BN, BL::kContigK>;
  constexpr int GPT = BN * 8;                         // float4 groups per tile (BN rows x 32 floats)
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)ntn * ktiles * GPT) return;
  const int tile = (int)(g / GPT), lg = (int)(g % GPT);
  const int nt = tile / ktiles, kt = tile - nt * ktiles;
  int n, k, off;
  if (BL::kContigK) {
    const int r = lg >> 3, kq = lg & 7;
    n = nt * BN + r; k = kt * 32 + kq * 4; off = TB::chunk_off(r, kq * 4);
  } else {
    const int q = lg % (BN / 4), kk = lg / (BN / 4);
    n = nt * BN + q * 4; k = kt * 32 + kk; off = TB::chunk_off(q * 4, kk);
  }
  const typename BL::Row row = bl.row(0, n < N ? n : -1);
  const float4 v = (k < K) ? bl.load(row, k) : zero4();
  float4 h, l;
  umma::split4(v, h, l);
  uint8_t* dst = image + (size_t)tile * (2 * TB::BYTES);
  TB::put(dst, off, h);
  TB::put(dst + TB::BYTES, off, l);
}

template <int BN>
inline size_t weight_image_bytes(int N, int K) {
  return (size_t)cdiv(N, BN) * cdiv(K, 32) * 2 * BN * 128;
}

template <int BN, class BL>
inline int launch_retile_b(cudaStream_t s, const BL& bl, int N, int K, uint8_t* image) {
  const int ntn = cdiv(N, BN), ktiles = cdiv(K, 32);
  const long long groups = (long long)ntn * ktiles * BN * 8;
  DRL_CUDA_CHECK((launch_k(retile_b_kernel<BN, BL>, (unsigned)cdiv64(groups, 256), 256, 0, s, bl, N, K, ktiles, ntn, image)));
  return DRL_OK;
}

template <class Cfg, class AL, class BL, class EP>
inline int launch_gemm_umma(cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                            int zcount, int kchunk, int kstep) {
  using SM = UmmaSmem<Cfg, AL, BL>;
  static bool attr_done = false;
  auto kern = gemm_umma_kernel<Cfg, AL, BL, EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::BYTES));
    attr_done = true;
  }
  if ((AL::kContigK || BL::kContigK) && (K % 4 != 0 || kchunk % 4 != 0)) {
    set_error("gemm_umma: K (%d) and kchunk (%d) must be multiples of 4 for K-contiguous operands", K, kchunk);
    return DRL_ERR_INVALID;
  }
  if (kchunk < 1 || K < 1) { set_error("gemm_umma: empty K range"); return DRL_ERR_INVALID; }
  static_assert(Cfg::STAGES >= 2, "consumers hand a stage back only after the next stage's MMAs are issued");
  dim3 grid(cdiv(M, Cfg::BM), cdiv(N, Cfg::BN), zcount);
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT, SM::BYTES, s, al, bl, ep, M, N, K, kchunk, kstep)));
  return DRL_OK;
}

}  // namespace drl
