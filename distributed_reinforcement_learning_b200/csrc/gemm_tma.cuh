// gemm_tma.cuh -- TMA-fed wgmma convolution forward (conv2 / conv3 of model/impala_actor_critic.py:7-8).
//
// The software-producer core (gemm_umma.cuh) spends its time in the LSU pipe: every A element is fetched with LDG,
// split into hi/lo in registers and written to shared memory with STS.  For the NHWC convolutions this im2col
// gather can be described to the TMA engine exactly, because one K tile (32 input channels of ONE filter tap) of
// one whole image is a 4-D box of the activation tensor:
//
//     tap (kh, kw):  base = act + ((kh*IH + kw)*CIN) floats
//                    dims {CIN, OH, OH, images, plane}, strides {S*CIN, S*IH*CIN, IH*IH*CIN, plane} floats
//                    box  {32, OH, OH, IMGS, 1}  ->  IMGS*OH*OH rows of 128 bytes, written with SWIZZLE_128B:
//                    byte for byte the K-major wgmma operand tile (rows = output pixels of IMGS whole images).
//
// The hi/lo split of 3xTF32 is done by the PRODUCING kernel's epilogue instead: plane 0 is the activation itself
// (the tensor core reads the upper 19 bits of each 32-bit word, i.e. hi = trunc_tf32(x)), plane 1 holds
// lo = x - trunc_tf32(x), exact in fp32.  A_lo*B_hi + A_hi*B_lo + A_hi*B_hi then drops only lo*lo ~ 2^-20.
// The weights come from the pre-split, pre-tiled image of retile_b_kernel (one cp.async.bulk per K tile).
//
// One CTA per SM, persistent over tiles of IMGS whole images (rows beyond IMGS*OH*OH of the 128-row MMA are
// ignored by the epilogue):
//   warps 0..5  TMA producers (one lane each): per K tile two tensor loads (planes 0/1) + one bulk copy, each issued
//               by its own warp with arrive.expect_tx on full[stage]; two groups of three warps alternate K tiles
//               (warps 6, 7 idle: the consumers start on a warpgroup boundary)
//   warps 8..15 two consumer warpgroups (rows 0-63 / 64-127): 12 wgmma per K tile into the register accumulator,
//               stage hand-back (empty), then bias + ReLU and coalesced stores of the activation and its lo plane (the
//               next layer's TMA operand) while the producers already load the next tile
#pragma once
#include <cuda.h>

#include <map>
#include <tuple>

#include "gemm_umma_persist.cuh"

namespace drl {

namespace umma {
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            int c4, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4),
      "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
}  // namespace umma

// geometry of one TMA-fed convolution layer
template <int CIN_, int IH_, int OH_, int KS_, int STRIDE_, int IMGS_, int NSTAGE_>
struct ConvTmaCfg {
  static constexpr int CIN = CIN_, IH = IH_, OH = OH_, KS = KS_, STRIDE = STRIDE_, IMGS = IMGS_, NSTAGE = NSTAGE_;
  static constexpr int BN = 64;                          // output channels (both layers)
  static constexpr int TAPS = KS * KS, HALVES = CIN / 32, NKT = TAPS * HALVES;
  static constexpr int PIX = OH * OH, ROWS = PIX * IMGS; // valid rows of the 128-row tile
  static_assert(ROWS <= 128 && CIN % 32 == 0, "tile = whole images, K tile = 32 channels of one tap");
  static constexpr int A_BYTES = 128 * 128, B_BYTES = BN * 128;
  static constexpr int BOX_BYTES = ROWS * 128;           // bytes one tensor load delivers
  static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
  static constexpr int PGROUPS = 2, PWARPS = 3 * PGROUPS;   // producer warps (one issuing lane each)
  static constexpr int CW0 = 8;                          // first consumer warp (warpgroup aligned)
  static constexpr int NT = CW0 * 32 + wg::kConsumerThreads;
  static constexpr int AUX_BYTES = 1024;
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + AUX_BYTES + 8 * wg::kEpiWarpBytes + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory");
};

template <int TAPS>
struct ConvTmaMaps {
  CUtensorMap tap[TAPS];
};

template <class Cfg, class EP>
__global__ void __launch_bounds__(Cfg::NT, 1)
conv_fwd_tma_kernel(const __grid_constant__ ConvTmaMaps<Cfg::TAPS> maps, const uint8_t* __restrict__ wimage, const EP ep,
                    int nimg, int ntiles) {
  pdl_prologue();
  constexpr int NSTAGE = Cfg::NSTAGE, NKT = Cfg::NKT, BN = Cfg::BN;
  using TA = UmmaTile<128, true>;
  using TB = UmmaTile<BN, false>;    // the weight image of a [K, N] row-major matrix (stored K-major by retile_b_kernel)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* aux = smem + NSTAGE * Cfg::STAGE_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(aux);
  uint64_t* empty = full + NSTAGE;
  uint8_t* stg_base = aux + Cfg::AUX_BYTES;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      umma::mbar_init(&full[s], 3);     // hi plane, lo plane, weight tile: one arrive.expect_tx each
      umma::mbar_init(&empty[s], wg::kConsumerWGs);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();

  if (warp < Cfg::PWARPS) {
    // ================= TMA PRODUCERS =================
    // One cp.async.bulk(.tensor) costs its issuing thread ~0.24 us whatever its size (tools/microbench/tma_box_bw.cu),
    // so the three copies of a K tile are issued by three different warps, and two such groups alternate K tiles.
    if (lane == 0) {
      const int group = warp / 3, role = warp % 3;
      if (role < 2)
        for (int t = 0; t < Cfg::TAPS; ++t) umma::prefetch_tensormap(&maps.tap[t]);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int img0 = tile * Cfg::IMGS;
        for (int kt = 0; kt < NKT; ++kt, ++it) {
          if ((int)(it % Cfg::PGROUPS) != group) continue;
          const int s = it % NSTAGE;
          umma::mbar_wait(&empty[s], ((it / NSTAGE) & 1) ^ 1);
          uint8_t* st = smem + s * Cfg::STAGE_BYTES;
          if (role < 2) {
            umma::mbar_arrive_expect_tx(&full[s], Cfg::BOX_BYTES);
            umma::tma_load_5d(st + role * Cfg::A_BYTES, &maps.tap[kt / Cfg::HALVES], (kt % Cfg::HALVES) * 32, 0, 0, img0,
                              role, &full[s]);
          } else {
            umma::mbar_arrive_expect_tx(&full[s], 2 * Cfg::B_BYTES);
            umma::bulk_g2s(st + 2 * Cfg::A_BYTES, wimage + (size_t)kt * (2 * Cfg::B_BYTES), 2 * Cfg::B_BYTES, &full[s]);
          }
        }
      }
    }
  } else if (warp >= Cfg::CW0) {
    // ================= CONSUMERS (warpgroup cw = rows 64 cw .. 64 cw + 63 of the tile) =================
    const int ct = tid - Cfg::CW0 * 32, cw = ct >> 7, cwarp = (ct >> 5) & 3;
    uint8_t* stg = stg_base + (ct >> 5) * wg::kEpiWarpBytes;
    uint32_t it = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      for (int kt = 0; kt < NKT; ++kt, ++it) {
        const int s = it % NSTAGE;
        umma::mbar_wait(&full[s], (it / NSTAGE) & 1);
        const uint32_t st = umma::smem_u32(smem + s * Cfg::STAGE_BYTES);
        const uint32_t a_hi = st + cw * 64 * 128, b_hi = st + 2 * Cfg::A_BYTES;
        wg::fence_operand(acc);
        wg::fence();
        tf32_stage_mmas<BN, false, 32, TA, TB>(acc, a_hi, a_hi + Cfg::A_BYTES, b_hi, b_hi + Cfg::B_BYTES, kt == 0);
        wg::commit();
        wg::wait<1>();
        wg::fence_operand(acc);
        if (kt > 0 && (ct & 127) == 0) umma::mbar_arrive(&empty[(it - 1) % NSTAGE]);
      }
      wg::wait<0>();
      wg::fence_operand(acc);
      if ((ct & 127) == 0) umma::mbar_arrive(&empty[(it - 1) % NSTAGE]);
      const int row_base = tile * Cfg::IMGS * Cfg::PIX;
      const int row_end = min(nimg * Cfg::PIX, row_base + Cfg::ROWS);
      wg_epilogue<BN>(ep, acc, stg, lane, 0, row_base + cw * 64 + cwarp * 16, 0, row_end, BN);
    }
  }
}

// ---- host side -------------------------------------------------------------------------------
typedef CUresult (*TmaEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline TmaEncodeTiledFn tma_encode_fn() {
  static TmaEncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<TmaEncodeTiledFn>(p);
  }();
  return fn;
}

// act: plane 0 of the NHWC activation [nimg, IH, IH, CIN]; plane 1 (lo) starts plane_floats later
template <class Cfg>
inline int conv_tma_maps(const float* act, size_t plane_floats, int nimg, ConvTmaMaps<Cfg::TAPS>* out) {
  TmaEncodeTiledFn enc = tma_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available in this driver"); return DRL_ERR_CUDA; }
  for (int kh = 0; kh < Cfg::KS; ++kh)
    for (int kw = 0; kw < Cfg::KS; ++kw) {
      const float* base = act + (size_t)(kh * Cfg::IH + kw) * Cfg::CIN;
      const cuuint64_t dims[5] = {(cuuint64_t)Cfg::CIN, (cuuint64_t)Cfg::OH, (cuuint64_t)Cfg::OH, (cuuint64_t)nimg, 2};
      const cuuint64_t strides[4] = {(cuuint64_t)Cfg::STRIDE * Cfg::CIN * 4, (cuuint64_t)Cfg::STRIDE * Cfg::IH * Cfg::CIN * 4,
                                     (cuuint64_t)Cfg::IH * Cfg::IH * Cfg::CIN * 4, (cuuint64_t)plane_floats * 4};
      const cuuint32_t box[5] = {32, (cuuint32_t)Cfg::OH, (cuuint32_t)Cfg::OH, (cuuint32_t)Cfg::IMGS, 1};
      const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
      const CUresult r = enc(&out->tap[kh * Cfg::KS + kw], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base),
                             dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) for tap %d,%d", (int)r, kh, kw); return DRL_ERR_CUDA; }
    }
  return DRL_OK;
}

template <class Cfg, class EP>
inline int launch_conv_fwd_tma(cudaStream_t s, const float* act, size_t plane_floats, int nimg, const uint8_t* wimage,
                               const EP& ep) {
  // the maps depend only on (activation pointer, plane stride, image count): encode once, reuse
  using Key = std::tuple<const float*, size_t, int>;
  static thread_local std::map<Key, ConvTmaMaps<Cfg::TAPS>> cache;
  const Key key{act, plane_floats, nimg};
  auto it = cache.find(key);
  if (it == cache.end()) {
    ConvTmaMaps<Cfg::TAPS> m;
    DRL_TRY((conv_tma_maps<Cfg>(act, plane_floats, nimg, &m)));
    it = cache.emplace(key, m).first;
  }
  static bool attr_done = false;
  auto kern = conv_fwd_tma_kernel<Cfg, EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done = true;
  }
  const int ntiles = cdiv(nimg, Cfg::IMGS);
  const int grid = std::min(ntiles, device_sm_count());
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT, Cfg::SMEM_BYTES, s, it->second, wimage, ep, nimg, ntiles)));
  return DRL_OK;
}

}  // namespace drl
