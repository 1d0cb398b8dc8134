// gemm_bulk16.cuh -- wgmma GEMM whose BOTH operands are pre-tiled 16-bit images: no producer warps at all.
//
// The gather-GEMMs of gemm_umma16.cuh feed the tensor core through producer warps (LDG fp32 -> split into bf16 hi/lo ->
// STS).  For the three LSTM contractions of model/impala_actor_critic.py:18-25 (forward z = [a3|emb|h0] W, data
// gradient dx = dz W^T, weight gradient dW = x^T dz) that path, not the MMAs, set the pace: 32 KB of A per K tile took
// the eight producer warps ~3 us, while the 64 KB weight tile next to it arrived by ONE cp.async.bulk in a fraction of
// that.  Here the activation-side operand is ALSO written once as an image (retile_b16_kernel over the activation
// loader: x as rows x K, x^T, dz, dz^T -- 2.4-9.3 MB each, written once, read by 4-29 CTAs each), so a K tile of a CTA is
// two bulk copies that complete on the stage's mbarrier (expect_tx) and twelve wgmma per consumer warpgroup:
//
//     image tile (row tile rt, k tile kt) = [hi plane | lo plane], each ROWS x 128 bytes K-major SWIZZLE_128B
//     (byte for byte what a stage holds; Umma16Tile<ROWS, true>), at image + (rt * ktiles + kt) * 2 * ROWS * 128
//
//   warp 0      loader: one lane, per K tile arrive.expect_tx + 2 bulk copies (A tile 32 KB, B tile BN x 256 B)
//               (warps 1-3 idle: the consumers must start on a warpgroup boundary)
//   warps 4-11  two consumer warpgroups (rows 0-63 / 64-127): MMA issue (A_lo B_hi + A_hi B_lo + A_hi B_hi per K = 16
//               slice) into the register accumulator, stage hand-back (empty), then the epilogue through the dead
//               stages (wg_epilogue)
// Rows beyond M / N and k beyond K are zero in the images, so no masking is needed before the epilogue.
#pragma once
#include "gemm_umma16.cuh"

namespace drl {

template <int BN_, int STAGES_>
struct Bulk16Cfg {
  static constexpr int BM = 128, BN = BN_, BK = 64, STAGES = STAGES_;
  static constexpr int NT = 128 + wg::kConsumerThreads;                  // loader warpgroup + two consumer warpgroups
  static constexpr int A_BYTES = BM * 128, B_BYTES = BN * 128;            // one plane
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 1024;   // stages + barriers + alignment
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN must be a power of two in [32,256]");
  static_assert(STAGES * STAGE_BYTES >= 8 * wg::kEpiWarpBytes, "epilogue staging tiles live in the dead stages");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

struct ImageOp {
  const uint8_t* image;
  int ktiles;   // K tiles per row tile in the image
};

template <class Cfg, class EP>
__global__ void __launch_bounds__(Cfg::NT, 1)
gemm_bulk16_kernel(const ImageOp a, const ImageOp b, const EP ep, int M, int N, int K, int kchunk, int kstep) {
  kernel_prologue();
  const Trace16 TR = trace16_arm();   // tools/umma16_timeline.py: same tags as gemm_umma16_kernel
  if (threadIdx.x == 0) TR((1ull << 40) | ((unsigned long long)gridDim.x << 20) | (gridDim.y * gridDim.z * 1024 + (Cfg::BN & 1023)));
  constexpr int BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES;
  using TA = Umma16Tile<128, true>;
  using TB = Umma16Tile<BN, true>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* aux = smem + STAGES * Cfg::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty = full + STAGES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int z = blockIdx.z;
  const int m0 = blockIdx.x * 128, n0 = blockIdx.y * BN;
  const int k0 = z * kstep;                       // multiple of 64 (checked by the launcher)
  const int k1 = min(K, k0 + kchunk);
  const int ntiles = (k1 - k0 + BK - 1) / BK;
  const int kt0 = k0 / BK;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      umma::mbar_init(&full[s], 1);
      umma::mbar_init(&empty[s], wg::kConsumerWGs);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) TR(2);

  if (warp == 0) {
    // ================= LOADER =================
    if (lane == 0) {
      const uint8_t* asrc = a.image + ((size_t)blockIdx.x * a.ktiles + kt0) * (size_t)(2 * Cfg::A_BYTES);
      const uint8_t* bsrc = b.image + ((size_t)blockIdx.y * b.ktiles + kt0) * (size_t)(2 * Cfg::B_BYTES);
      for (int t = 0; t < ntiles; ++t) {
        const int s = t % STAGES;
        umma::mbar_wait(&empty[s], ((t / STAGES) & 1) ^ 1);
        uint8_t* st = smem + s * Cfg::STAGE_BYTES;
        TR(5000 + t);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(&full[s])),
                     "r"(Cfg::STAGE_BYTES) : "memory");
        umma::bulk_g2s(st, asrc + (size_t)t * (2 * Cfg::A_BYTES), 2 * Cfg::A_BYTES, &full[s]);
        umma::bulk_g2s(st + 2 * Cfg::A_BYTES, bsrc + (size_t)t * (2 * Cfg::B_BYTES), 2 * Cfg::B_BYTES, &full[s]);
      }
    }
  } else if (warp >= 4) {
    // ================= CONSUMERS (warps 4..11: warpgroup cw = rows 64 cw .. 64 cw + 63) =================
    const int ct = tid - 128, cw = ct >> 7, cwarp = (ct >> 5) & 3;
    const uint64_t da_base = umma::make_desc(0, TA::LBO, TA::SBO), db_base = umma::make_desc(0, TB::LBO, TB::SBO);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int t = 0; t < ntiles; ++t) {
      const int s = t % STAGES;
      umma::mbar_wait(&full[s], (t / STAGES) & 1);
      if (ct == 0) TR(3000 + t);
      const uint32_t st = umma::smem_u32(smem + s * Cfg::STAGE_BYTES);
      const uint64_t a_hi = umma::desc_at(da_base, st + cw * 64 * 128);
      const uint64_t a_lo = umma::desc_at(da_base, st + Cfg::A_BYTES + cw * 64 * 128);
      const uint64_t b_hi = umma::desc_at(db_base, st + 2 * Cfg::A_BYTES);
      const uint64_t b_lo = umma::desc_at(db_base, st + 2 * Cfg::A_BYTES + Cfg::B_BYTES);
      wg::fence_operand(acc);
      wg::fence();
#pragma unroll
      for (int j = 0; j < BK / 16; ++j) {
        const uint64_t ao = (uint64_t)(TA::kslice_off(j) >> 4), bo = (uint64_t)(TB::kslice_off(j) >> 4);
        umma16::mma16<BN, umma16::BF16, 0, 0>(acc, a_lo + ao, b_hi + bo, (t > 0 || j > 0) ? 1u : 0u);   // small terms first
        umma16::mma16<BN, umma16::BF16, 0, 0>(acc, a_hi + ao, b_lo + bo, 1u);
        umma16::mma16<BN, umma16::BF16, 0, 0>(acc, a_hi + ao, b_hi + bo, 1u);
      }
      wg::commit();
      wg::wait<1>();
      wg::fence_operand(acc);
      if (t > 0 && (ct & 127) == 0) umma::mbar_arrive(&empty[(t - 1) % STAGES]);
      if (ct == 0) TR(4000 + t);
    }
    wg::wait<0>();
    wg::fence_operand(acc);
    // ================= EPILOGUE =================
    wg::consumer_sync();                               // all stages are dead once both accumulators are complete
    if (ct == 0) TR(6000);
    uint8_t* stg = smem + (ct >> 5) * wg::kEpiWarpBytes;
    wg_epilogue<BN>(ep, acc, stg, lane, z, m0 + cw * 64 + cwarp * 16, n0, M, N);
    if (ct == 0) TR(6001);
  }
}

template <class Cfg, class EP>
inline int launch_gemm_bulk16(cudaStream_t s, const ImageOp& a, const ImageOp& b, const EP& ep, int M, int N, int K,
                              int zcount, int kchunk, int kstep) {
  static bool attr_done = false;   // per instantiation
  auto kern = gemm_bulk16_kernel<Cfg, EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done = true;
  }
  if (kstep % 64 != 0 || (zcount > 1 && kchunk % 64 != 0)) {
    set_error("gemm_bulk16: split-K offsets (kstep %d, kchunk %d) must be multiples of the 64-element K tile", kstep, kchunk);
    return DRL_ERR_INVALID;
  }
  dim3 grid(cdiv(M, 128), cdiv(N, Cfg::BN), zcount);
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT, Cfg::SMEM_BYTES, s, a, b, ep, M, N, K, kchunk, kstep)));
  return DRL_OK;
}

// bytes of the image of a [rows x K] operand in ROWS-row tiles
template <int ROWS>
inline size_t operand_image16_bytes(int rows, int K) {
  return (size_t)cdiv(rows, ROWS) * cdiv(K, 64) * 2 * ROWS * 128;
}

}  // namespace drl
