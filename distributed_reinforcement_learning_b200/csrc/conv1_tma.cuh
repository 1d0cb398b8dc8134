// conv1_tma.cuh -- conv1 of the attention_CNN (model/impala_actor_critic.py:6: 8x8 stride 4 over 84x84x4 uint8 frames ->
// 20x20x32, ReLU) as a FRAME-RESIDENT, TMA-fed, warp-specialised wgmma kernel (math mode 5).
//
// The generic gather-GEMM spends conv1's time in per-CTA fixed costs: 2000 CTAs of one 128-row tile each (K = 256 only),
// every one paying barrier set-up, a cold first gather and a serial epilogue, and every frame byte is gathered 4x
// through the LSU (8x8 windows at stride 4 overlap).  Here one persistent CTA per SM walks over whole frames:
//
//   TMA warp      one tensor load per frame: the raw 84x84x4 bytes (28,224 B) -> shared memory, double-buffered
//                 (tensor map {16 B, 21, 84, frames}, box = one frame; the (t,b) -> b*T+t remap of the caller's batch-major
//                 trajectory buffer is just the box coordinate)
//   8 converter   expand the im2col FROM SHARED MEMORY: a task (pixel, ky) reads the 32 contiguous bytes of one window row,
//   warps         turns them into 32 fp16 (exact: PRMT + HSUB2) and writes 4 swizzled 16-byte chunks of a K-major
//                 SWIZZLE_128B operand stage [128 pixels x 64 features]; 16 stages per frame (4 M tiles x 4 K chunks)
//                 through a ring of 6; four groups of two warps, group g owns chunk g (4 tasks per thread and stage)
//   consumer      one warpgroup (warps 8-11): per stage 2 x 4 wgmma (f16, M64 N64 K16) for the two 64-pixel halves of the
//   warpgroup     tile; the B tile is [W_hi ; W_lo] stacked along N (the two planes of the weight image are adjacent, i.e.
//                 ONE 64-row K-major tile), so A x W_hi lands in columns 0-31 and A x W_lo in columns 32-63 of the
//                 register accumulator and the epilogue adds the halves -- half the instructions of issuing the two
//                 products separately.  After the 4 stages of a tile: /255 (true fp32 divide, agent/impala.py:133) + bias
//                 + ReLU -> coalesced stores of the a1 rows, while the converters already fill the ring for the next tile
//
// Algorithmic traffic per frame: 28,224 B read once (TMA) + 51,200 B of a1 written; shared memory sees the 4x im2col
// amplification instead of L2 (102 KB read, 205 KB written, 205 KB read by the tensor core per frame).
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include <map>
#include <tuple>

#include "gemm_umma16.cuh"
#include "gemm_umma_persist.cuh"
#include "loaders.cuh"

namespace drl {

namespace umma {
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
}  // namespace umma

struct Conv1Tma {
  static constexpr int FRAME = Geo::FRAME;            // 28,224 bytes
  static constexpr int PIX = Geo::C1H * Geo::C1W;     // 400 output pixels per frame
  static constexpr int MT = 4;                        // 128-row M tiles per frame (the last one holds 16 pixels)
  static constexpr int KC = 4;                        // K chunks of 64 features (two window rows ky) per M tile
  static constexpr int NS = 6;                        // operand stages in the ring
  static constexpr int STAGE_BYTES = 128 * 128;       // 128 pixels x 64 fp16
  static constexpr int RAW_STRIDE = 28672;            // frame buffer pitch (128-byte multiple)
  static constexpr int W_BYTES = 4 * 2 * 32 * 128;    // 4 K tiles x [hi | lo] x 32 rows x 128 B = 32 KB
  static constexpr int CONV_WARPS = 8, EPI_WARPS = 4;
  static constexpr int W_TMA = CONV_WARPS + EPI_WARPS;   // warps 0-7 convert, 8-11 MMA + epilogue (one warpgroup), 12 TMA
  static constexpr int NT = (W_TMA + 1) * 32;         // 416 threads
  static constexpr int OFF_RAW = NS * STAGE_BYTES;
  static constexpr int OFF_W = OFF_RAW + 2 * RAW_STRIDE;
  static constexpr int OFF_EPI = OFF_W + W_BYTES;
  static constexpr int OFF_AUX = OFF_EPI + EPI_WARPS * wg::kEpiWarpBytes;
  static constexpr int OFF_DBG = OFF_AUX + 512;        // 4 roles x 96 clock samples (debug timeline, tools/conv1_timeline.py)
  static constexpr int SMEM_BYTES = OFF_DBG + 4 * 96 * 8 + 1024;
};

template <class EP>
__global__ void __launch_bounds__(Conv1Tma::NT, 1)
conv1_fwd_tma_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ wf32, const EP ep, RowMap map,
                     int nframes) {
  kernel_prologue();
  using C = Conv1Tma;
  using TA = Umma16Tile<128, true>;
  using TB = Umma16Tile<32, true>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* raw = smem + C::OFF_RAW;
  uint8_t* wsm = smem + C::OFF_W;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + C::OFF_AUX);   // [NS]
  uint64_t* a_empty = a_full + C::NS;                                  // [NS]
  uint64_t* raw_full = a_empty + C::NS;                                // [2]
  uint64_t* raw_empty = raw_full + 2;                                  // [2]
  uint64_t* w_full = raw_empty + 2;                                    // [1]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // debug timeline: when the trace buffer is armed with magic 0xC0171 in word 8001, lane 0 of each role keeps clock64()
  // samples in shared memory (no global traffic while running) and CTA 0 dumps them behind word 8002 at the end
  long long* dbg = reinterpret_cast<long long*>(smem + C::OFF_DBG);
  unsigned long long* const trbuf = g_trace_tu;
  const bool tracing = trbuf != nullptr && trbuf[8001] == 0xC0171ull && blockIdx.x == 0;
  int dn = 0;
#define C1_TR(role) do { if (tracing && dn < 96) dbg[(role) * 96 + dn++] = clock64(); } while (0)
  if (tracing) for (int i = tid; i < 4 * 96; i += blockDim.x) dbg[i] = 0;
  if (tid == 0) {
    for (int s = 0; s < C::NS; ++s) {
      umma::mbar_init(&a_full[s], C::CONV_WARPS * 32 / 4);   // one converter group (2 warps) per stage
      umma::mbar_init(&a_empty[s], 1);
    }
    for (int b = 0; b < 2; ++b) {
      umma::mbar_init(&raw_full[b], 1);
      umma::mbar_init(&raw_empty[b], C::CONV_WARPS * 32);
    }
    // weights: the epilogue warps build the image from the fp32 HWIO weights themselves while the first frame slab is in
    // flight: the step's first kernel then has no weight-image kernel in front of it (5 us at the head of every step)
    umma::mbar_init(w_full, C::EPI_WARPS * 32);
    umma::fence_barrier_init();
  }
  __syncthreads();

  if (warp < C::CONV_WARPS) {
    // ================= CONVERTERS: raw frame bytes -> fp16 K-major operand stages =================
    // Four groups of two warps; group g builds K chunk g (window rows 2g, 2g+1) of every M tile on its own, four
    // (pixel, window row) tasks per thread and ONE fence + arrive per thread and stage: the per-stage barrier / fence latency
    // (measured ~450 of ~550 cycles per stage when every thread took part in every stage) is paid a quarter as often
    // per thread and the four chunks of a tile are converted concurrently.
    const int g = tid >> 6, lt = tid & 63;
    int fi = 0;
    uint32_t tile = 0;
    for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x, ++fi) {
      const int slot = fi & 1;
      umma::mbar_wait(&raw_full[slot], (fi >> 1) & 1);
      const uint8_t* fr = raw + slot * C::RAW_STRIDE;
#pragma unroll 1
      for (int mt = 0; mt < C::MT; ++mt, ++tile) {
        const uint32_t it = tile * C::KC + g;          // stage counter of (tile, chunk g)
        const int s = it % C::NS;
        // raw bytes of the four tasks first (independent of the stage barrier)
        uint4 r[4][2];
        bool live[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int p_local = lt + 64 * (q >> 1), kyl = q & 1;
          const int p = mt * 128 + p_local;
          live[q] = p < C::PIX;
          const int pc = live[q] ? p : 0;
          const int oy = pc / Geo::C1W, ox = pc - oy * Geo::C1W;
          const uint4* src = reinterpret_cast<const uint4*>(fr + (4 * oy + 2 * g + kyl) * (Geo::IW * Geo::IC) + 16 * ox);
          r[q][0] = src[0];
          r[q][1] = src[1];
        }
        umma::mbar_wait(&a_empty[s], ((it / C::NS) & 1) ^ 1);
        if (lt == 0 && g == 0) C1_TR(0);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (!live[q]) continue;
          const int p_local = lt + 64 * (q >> 1), kyl = q & 1;
          uint8_t* row = smem + s * C::STAGE_BYTES + p_local * 128;
          const int sw = p_local & 7, q0 = kyl * 4;
          uint2 h;
          uint4 o;
          h = umma16::u8x4_to_h4(r[q][0].x); o.x = h.x; o.y = h.y; h = umma16::u8x4_to_h4(r[q][0].y); o.z = h.x; o.w = h.y;
          *reinterpret_cast<uint4*>(row + (((q0 + 0) ^ sw) << 4)) = o;
          h = umma16::u8x4_to_h4(r[q][0].z); o.x = h.x; o.y = h.y; h = umma16::u8x4_to_h4(r[q][0].w); o.z = h.x; o.w = h.y;
          *reinterpret_cast<uint4*>(row + (((q0 + 1) ^ sw) << 4)) = o;
          h = umma16::u8x4_to_h4(r[q][1].x); o.x = h.x; o.y = h.y; h = umma16::u8x4_to_h4(r[q][1].y); o.z = h.x; o.w = h.y;
          *reinterpret_cast<uint4*>(row + (((q0 + 2) ^ sw) << 4)) = o;
          h = umma16::u8x4_to_h4(r[q][1].z); o.x = h.x; o.y = h.y; h = umma16::u8x4_to_h4(r[q][1].w); o.z = h.x; o.w = h.y;
          *reinterpret_cast<uint4*>(row + (((q0 + 3) ^ sw) << 4)) = o;
        }
        umma::fence_proxy_async();
        umma::mbar_arrive(&a_full[s]);
        if (lt == 0 && g == 0) C1_TR(0);
      }
      umma::mbar_arrive(&raw_empty[slot]);        // this thread no longer reads the frame buffer
    }
  } else if (warp < C::W_TMA) {
    // ================= MMA + EPILOGUE (warps 8..11: one warpgroup) =================
    const int cwarp = warp & 3;
    uint8_t* stg = smem + C::OFF_EPI + cwarp * wg::kEpiWarpBytes;
    // [K = 256][N = 32] fp32 -> per K tile of 64: rows 0..31 = fp16(w), rows 32..63 = fp16(w - hi) (K-major, swizzled):
    // 1024 units of 8 consecutive k of one n; lanes = consecutive n (coalesced 128-byte rows of the HWIO matrix)
    for (int u = tid - C::CONV_WARPS * 32; u < 32 * 32; u += C::EPI_WARPS * 32) {
      const int n = u & 31, kb = (u >> 5) * 8;
      float x[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) x[i] = __ldg(wf32 + (size_t)(kb + i) * 32 + n);
      uint4 h, l;
      umma16::split8<umma16::F16>(make_float4(x[0], x[1], x[2], x[3]), make_float4(x[4], x[5], x[6], x[7]), h, l);
      uint8_t* dst = wsm + (kb >> 6) * (2 * TB::BYTES);
      const int off = TB::chunk_off(n, kb & 63);
      *reinterpret_cast<uint4*>(dst + off) = h;
      *reinterpret_cast<uint4*>(dst + TB::BYTES + off) = l;
    }
    umma::fence_proxy_async();
    umma::mbar_arrive(w_full);
    umma::mbar_wait(w_full, 0);
    const uint64_t da_base = umma::make_desc(0, TA::LBO, TA::SBO), db_base = umma::make_desc(0, TB::LBO, TB::SBO);
    float acc0[32], acc1[32];   // pixels 0-63 / 64-127 of the tile x [A W_hi | A W_lo]
#pragma unroll
    for (int i = 0; i < 32; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    uint32_t it = 0;
    for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x) {
      const int row_base = mf * C::PIX, row_end = row_base + C::PIX;
      for (int mt = 0; mt < C::MT; ++mt) {
        for (int c = 0; c < C::KC; ++c, ++it) {
          const int s = it % C::NS;
          umma::mbar_wait(&a_full[s], (it / C::NS) & 1);
          if (cwarp == 0 && lane == 0) C1_TR(1);
          const uint32_t sa = umma::smem_u32(smem + s * C::STAGE_BYTES);
          const uint64_t a0 = umma::desc_at(da_base, sa), a1 = umma::desc_at(da_base, sa + 64 * 128);
          const uint64_t b = umma::desc_at(db_base, umma::smem_u32(wsm + c * (2 * TB::BYTES)));   // [W_hi ; W_lo]: 64 rows
          wg::fence_operand(acc0);
          wg::fence_operand(acc1);
          wg::fence();
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const uint64_t ko = (uint64_t)(j * 32 >> 4);
            umma16::mma16<64, umma16::F16, 0, 0>(acc0, a0 + ko, b + ko, (c > 0 || j > 0) ? 1u : 0u);
            umma16::mma16<64, umma16::F16, 0, 0>(acc1, a1 + ko, b + ko, (c > 0 || j > 0) ? 1u : 0u);
          }
          wg::commit();
          wg::wait<1>();                               // the MMAs of the previous stage are complete: hand it back
          wg::fence_operand(acc0);
          wg::fence_operand(acc1);
          if (c > 0 && tid == C::CONV_WARPS * 32) umma::mbar_arrive(&a_empty[(it - 1) % C::NS]);
        }
        wg::wait<0>();
        wg::fence_operand(acc0);
        wg::fence_operand(acc1);
        if (tid == C::CONV_WARPS * 32) umma::mbar_arrive(&a_empty[(it - 1) % C::NS]);
        if (cwarp == 0 && lane == 0) C1_TR(2);
        const int r0 = row_base + mt * 128 + cwarp * 16;
        wg_epilogue<64, true>(ep, acc0, stg, lane, 0, r0, 0, row_end, 32);
        wg_epilogue<64, true>(ep, acc1, stg, lane, 0, r0 + 64, 0, row_end, 32);
        if (cwarp == 0 && lane == 0) C1_TR(2);
      }
    }
  } else if (warp == C::W_TMA) {
    // ================= TMA PRODUCER =================
    if (lane == 0) {
      umma::prefetch_tensormap(&fmap);
      int fi = 0;
      for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x, ++fi) {
        const int slot = fi & 1;
        umma::mbar_wait(&raw_empty[slot], ((fi >> 1) & 1) ^ 1);
        C1_TR(3);
        umma::mbar_arrive_expect_tx(&raw_full[slot], C::FRAME);
        umma::tma_load_4d(raw + slot * C::RAW_STRIDE, &fmap, 0, 0, 0, map.src(mf), &raw_full[slot]);
      }
    }
  }
  __syncthreads();
  if (tracing) {
    for (int i = tid; i < 4 * 96; i += blockDim.x) trbuf[8002 + i] = (unsigned long long)dbg[i];
  }
#undef C1_TR
}

// ---- host side ---------------------------------------------------------------------------------------------------
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

// frames: the staging slot's uint8 [nframes, 84, 84, 4] buffer (caller's batch-major order)
inline int conv1_frame_map(const uint8_t* frames, int nframes, CUtensorMap* out) {
  TmaEncodeTiledFn enc = tma_encode_fn();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available in this driver"); return DRL_ERR_CUDA; }
  const cuuint64_t dims[4] = {16, 21, 84, (cuuint64_t)nframes};
  const cuuint64_t strides[3] = {16, 336, (cuuint64_t)Geo::FRAME};
  const cuuint32_t box[4] = {16, 21, 84, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<uint8_t*>(frames), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) for the frame map", (int)r); return DRL_ERR_CUDA; }
  return DRL_OK;
}

template <class EP>
inline int launch_conv1_fwd_tma(cudaStream_t s, const uint8_t* frames, int nframes, const RowMap& map, const float* wf32,
                                const EP& ep) {
  using Key = std::tuple<const uint8_t*, int>;
  static thread_local std::map<Key, CUtensorMap> cache;
  const Key key{frames, nframes};
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    DRL_TRY(conv1_frame_map(frames, nframes, &m));
    it = cache.emplace(key, m).first;
  }
  static bool attr_done = false;
  auto kern = conv1_fwd_tma_kernel<EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Conv1Tma::SMEM_BYTES));
    attr_done = true;
  }
  const int grid = std::min(nframes, device_sm_count());
  DRL_CUDA_CHECK((launch_k(kern, grid, Conv1Tma::NT, Conv1Tma::SMEM_BYTES, s, it->second, wf32, ep, map, nframes)));
  return DRL_OK;
}


// =====================================================================================================================
// conv1 weight gradient (the only gradient conv1 has: its input is data), same frame-resident scheme:
//     dW[f, n] = (1/255) sum_px X[px, f] dA1[px, n]      f = (ky, kx, ci) in [0, 256),  n in [0, 32),  px over Mb x 400
//     db[n]    = sum_px dA1[px, n]
//   TMA warp      per frame one tensor load of the raw bytes; per 64-pixel tile one bulk copy of the dA1 rows (8 KB fp32)
//   8 converter   A: the same im2col expansion as the forward, in bf16 (0..255 is exact in bf16 as well; bf16 because the
//   warps            other operand is a gradient): tile [64 px][256 features] as four K-major chunks = byte for byte the
//                    MN-major SWIZZLE_128B operand (M = feature contiguous, K = pixel) of the transposed product;
//                 B: dA1 [64 px][32] fp32 -> bf16 hi / lo, TRANSPOSED into one K-major tile of 64 rows [hi n | lo n] x 64 px
//                    (each thread: 8 consecutive pixels of one n = one 16-byte chunk per plane); column sums for db
//   2 consumer    warpgroup h (warps 8-11 / 12-15) owns features 128 h .. 128 h + 127: per tile 2 x 4 wgmma (bf16, M64
//   warpgroups    N64 K16, A MN-major, B K-major); the accumulators [X^T dA1_hi | X^T dA1_lo] stay in registers over ALL
//                 tiles of all frames of the CTA.  Once at the end: hi + lo halves, x 1/255, partial slab [257 x 32] of
//                 this CTA; a fixed-order reduce over the CTAs follows (splitk_reduce)
// =====================================================================================================================
struct Conv1WgTma {
  static constexpr int FRAME = Geo::FRAME, PIX = 400;
  static constexpr int TPX = 64;                       // pixels per tile
  static constexpr int NTILE = (PIX + TPX - 1) / TPX;  // 7 tiles per frame (the last one holds 16 pixels)
  static constexpr int A_SLOT = 4 * TPX * 128;         // 4 feature chunks x 64 px x 128 B = 32 KB
  static constexpr int B_SLOT = 64 * 128;              // 64 rows (32 hi + 32 lo) x 64 px bf16 = 8 KB
  static constexpr int D_SLOT = TPX * 32 * 4;          // raw dA1 rows of a tile, fp32: 8 KB
  static constexpr int RAW_STRIDE = 28672;
  static constexpr int CONV_WARPS = 8, MMA_WARPS = 8;
  static constexpr int W_TMA = CONV_WARPS + MMA_WARPS;   // warps 0-7 convert, 8-15 two consumer warpgroups, 16 TMA
  static constexpr int NT = (W_TMA + 1) * 32;
  static constexpr int OFF_B = 2 * A_SLOT;
  static constexpr int OFF_RAW = OFF_B + 2 * B_SLOT;
  static constexpr int OFF_D = OFF_RAW + 2 * RAW_STRIDE;
  static constexpr int OFF_AUX = OFF_D + 2 * D_SLOT;
  static constexpr int SMEM_BYTES = OFF_AUX + 512 + 1024;
  static constexpr int SLAB = 257 * 32;                // floats per CTA partial: dW [256 x 32] + db [32]
};

// 4 bytes -> 4 bf16 (exact): 2^23 + b as a float, minus 2^23, upper halves
__device__ __forceinline__ uint2 u8x4_to_bf4(uint32_t w) {
  const float m = 8388608.0f;
  const uint32_t f0 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7650)) - m);
  const uint32_t f1 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7651)) - m);
  const uint32_t f2 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7652)) - m);
  const uint32_t f3 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7653)) - m);
  return make_uint2(__byte_perm(f0, f1, 0x7632), __byte_perm(f2, f3, 0x7632));
}

static __global__ void __launch_bounds__(Conv1WgTma::NT, 1)
conv1_wgrad_tma_kernel(const __grid_constant__ CUtensorMap fmap, const float* __restrict__ da1, float* __restrict__ partial,
                       RowMap map, int nframes) {
  kernel_prologue();
  using C = Conv1WgTma;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bsm = smem + C::OFF_B;
  uint8_t* raw = smem + C::OFF_RAW;
  uint8_t* dsm = smem + C::OFF_D;
  uint64_t* t_full = reinterpret_cast<uint64_t*>(smem + C::OFF_AUX);   // [2] converted tile (A slot + B slot) ready
  uint64_t* t_empty = t_full + 2;                                      // [2]
  uint64_t* raw_full = t_empty + 2;                                    // [2]
  uint64_t* raw_empty = raw_full + 2;                                  // [2]
  uint64_t* d_full = raw_empty + 2;                                    // [2] raw dA1 rows of a tile
  uint64_t* d_empty = d_full + 2;                                      // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // operand slots start as zeros: rows of a partial tile keep stale (finite) values that meet zero B columns
  for (int i = tid; i < (C::OFF_RAW) / 16; i += blockDim.x) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (tid == 0) {
    for (int b = 0; b < 2; ++b) {
      umma::mbar_init(&t_full[b], C::CONV_WARPS * 32);
      umma::mbar_init(&t_empty[b], wg::kConsumerWGs);
      umma::mbar_init(&raw_full[b], 1);
      umma::mbar_init(&raw_empty[b], C::CONV_WARPS * 32);
      umma::mbar_init(&d_full[b], 1);
      umma::mbar_init(&d_empty[b], C::CONV_WARPS * 32);
    }
    umma::fence_barrier_init();
  }
  umma::fence_proxy_async();
  __syncthreads();
  float* slab = partial + (size_t)blockIdx.x * C::SLAB;

  if (warp < C::CONV_WARPS) {
    // ================= CONVERTERS =================
    const int pa = tid & 63, kyb = tid >> 6;            // A: pixel of the tile, window rows kyb and kyb + 4
    const int bn = tid >> 3, bj = tid & 7;              // B: column n, pixels 8 bj .. 8 bj + 7 of the tile
    float colsum = 0.f;
    uint32_t it = 0;
    int fi = 0;
    for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x, ++fi) {
      const int slot = fi & 1;
      umma::mbar_wait(&raw_full[slot], (fi >> 1) & 1);
      const uint8_t* fr = raw + slot * C::RAW_STRIDE;
#pragma unroll 1
      for (int pt = 0; pt < C::NTILE; ++pt, ++it) {
        const int ts = it & 1;
        const uint32_t ph = (it >> 1) & 1;
        umma::mbar_wait(&t_empty[ts], ph ^ 1);
        // ---- A: two window rows of this thread's pixel -> bf16 chunks of the feature chunks ky / 2
        const int p = pt * C::TPX + pa;
        if (p < C::PIX) {
          const int oy = p / Geo::C1W, ox = p - oy * Geo::C1W;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int ky = kyb + 4 * r;
            const uint4* src = reinterpret_cast<const uint4*>(fr + (4 * oy + ky) * (Geo::IW * Geo::IC) + 16 * ox);
            const uint4 r0 = src[0], r1 = src[1];
            uint8_t* row = smem + ts * C::A_SLOT + (ky >> 1) * (C::TPX * 128) + pa * 128;
            const int sw = pa & 7, q0 = (ky & 1) * 4;
            uint2 h;
            uint4 o;
            h = u8x4_to_bf4(r0.x); o.x = h.x; o.y = h.y; h = u8x4_to_bf4(r0.y); o.z = h.x; o.w = h.y;
            *reinterpret_cast<uint4*>(row + (((q0 + 0) ^ sw) << 4)) = o;
            h = u8x4_to_bf4(r0.z); o.x = h.x; o.y = h.y; h = u8x4_to_bf4(r0.w); o.z = h.x; o.w = h.y;
            *reinterpret_cast<uint4*>(row + (((q0 + 1) ^ sw) << 4)) = o;
            h = u8x4_to_bf4(r1.x); o.x = h.x; o.y = h.y; h = u8x4_to_bf4(r1.y); o.z = h.x; o.w = h.y;
            *reinterpret_cast<uint4*>(row + (((q0 + 2) ^ sw) << 4)) = o;
            h = u8x4_to_bf4(r1.z); o.x = h.x; o.y = h.y; h = u8x4_to_bf4(r1.w); o.z = h.x; o.w = h.y;
            *reinterpret_cast<uint4*>(row + (((q0 + 3) ^ sw) << 4)) = o;
          }
        }
        // ---- B: 8 consecutive pixels of column bn -> one 16-byte chunk of row bn (hi) and of row 32 + bn (lo)
        umma::mbar_wait(&d_full[ts], ph);
        {
          const float* d = reinterpret_cast<const float*>(dsm + ts * C::D_SLOT);
          float x[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int pl = 8 * bj + i;
            x[i] = (pt * C::TPX + pl < C::PIX) ? d[pl * 32 + bn] : 0.f;
            colsum += x[i];
          }
          uint4 hi, lo;
          umma16::split8<umma16::BF16>(make_float4(x[0], x[1], x[2], x[3]), make_float4(x[4], x[5], x[6], x[7]), hi, lo);
          uint8_t* bt = bsm + ts * C::B_SLOT;
          *reinterpret_cast<uint4*>(bt + bn * 128 + ((bj ^ (bn & 7)) << 4)) = hi;
          *reinterpret_cast<uint4*>(bt + (32 + bn) * 128 + ((bj ^ (bn & 7)) << 4)) = lo;
        }
        umma::mbar_arrive(&d_empty[ts]);
        umma::fence_proxy_async();
        umma::mbar_arrive(&t_full[ts]);
      }
      umma::mbar_arrive(&raw_empty[slot]);
    }
    // db: this thread summed column bn over pixels {8 bj .. 8 bj + 7} of every tile; the 8 threads of a column are lanes
    // 8k .. 8k+7 of one warp
    colsum += __shfl_xor_sync(0xffffffffu, colsum, 1);
    colsum += __shfl_xor_sync(0xffffffffu, colsum, 2);
    colsum += __shfl_xor_sync(0xffffffffu, colsum, 4);
    if (bj == 0) slab[256 * 32 + bn] = colsum;
  } else if (warp < C::W_TMA) {
    // ================= MMA (warpgroup h: features 128 h ..), epilogue once =================
    // A: MN-major (M = feature, K = pixel): atom = 8 px x 64 features = 1024 B; next 64 features = next chunk (LBO = 8 KB);
    //    next 8 pixels SBO = 1024; a K = 16 slice = 2 atoms = 2048 B.   B: K-major, 64 rows of 128 B.
    const int ct = tid - C::CONV_WARPS * 32, h = ct >> 7, cwarp = (ct >> 5) & 3;
    const uint64_t da_base = umma::make_desc(0, C::TPX * 128, 1024), db_base = umma::make_desc(0, 16, 1024);
    float acc0[32], acc1[32];   // features 128 h + [0, 64) / [64, 128) x [dA1_hi | dA1_lo]
#pragma unroll
    for (int i = 0; i < 32; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    uint32_t it = 0;
    for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x) {
      for (int pt = 0; pt < C::NTILE; ++pt, ++it) {
        const int ts = it & 1;
        umma::mbar_wait(&t_full[ts], (it >> 1) & 1);
        const uint64_t b = umma::desc_at(db_base, umma::smem_u32(bsm + ts * C::B_SLOT));
        const uint32_t sa = umma::smem_u32(smem + ts * C::A_SLOT + h * 2 * (C::TPX * 128));
        const uint64_t a0 = umma::desc_at(da_base, sa), a1 = umma::desc_at(da_base, sa + C::TPX * 128);
        wg::fence_operand(acc0);
        wg::fence_operand(acc1);
        wg::fence();
#pragma unroll
        for (int j = 0; j < C::TPX / 16; ++j) {
          const uint64_t ao = (uint64_t)(j * 2048 >> 4), bo = (uint64_t)(j * 32 >> 4);
          umma16::mma16<64, umma16::BF16, 1, 0>(acc0, a0 + ao, b + bo, (it > 0 || j > 0) ? 1u : 0u);
          umma16::mma16<64, umma16::BF16, 1, 0>(acc1, a1 + ao, b + bo, (it > 0 || j > 0) ? 1u : 0u);
        }
        wg::commit();
        wg::wait<1>();                                 // the previous tile's MMAs are complete: hand its slot back
        wg::fence_operand(acc0);
        wg::fence_operand(acc1);
        if (it > 0 && (ct & 127) == 0) umma::mbar_arrive(&t_empty[(it - 1) & 1]);
      }
    }
    wg::wait<0>();
    wg::fence_operand(acc0);
    wg::fence_operand(acc1);
    // fragment: acc[4c + e] = feature row lane/4 (+8 for e >= 2), column 8c + 2 (lane % 4) + (e & 1); c < 4: x dA1_hi,
    // c >= 4: the same column x dA1_lo
    const int r = lane >> 2, q = lane & 3;
#pragma unroll
    for (int sub = 0; sub < 2; ++sub) {
      const float* acc = sub ? acc1 : acc0;
      const int f0 = h * 128 + sub * 64 + cwarp * 16 + r;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int n = 8 * c + 2 * q, i = 4 * c;
        *reinterpret_cast<float2*>(slab + (size_t)f0 * 32 + n) =
            make_float2((acc[i] + acc[i + 16]) * (1.0f / 255.0f), (acc[i + 1] + acc[i + 17]) * (1.0f / 255.0f));
        *reinterpret_cast<float2*>(slab + (size_t)(f0 + 8) * 32 + n) =
            make_float2((acc[i + 2] + acc[i + 18]) * (1.0f / 255.0f), (acc[i + 3] + acc[i + 19]) * (1.0f / 255.0f));
      }
    }
  } else if (warp == C::W_TMA) {
    // ================= TMA PRODUCER =================
    if (lane == 0) {
      umma::prefetch_tensormap(&fmap);
      uint32_t it = 0;
      int fi = 0;
      for (int mf = blockIdx.x; mf < nframes; mf += gridDim.x, ++fi) {
        const int slot = fi & 1;
        umma::mbar_wait(&raw_empty[slot], ((fi >> 1) & 1) ^ 1);
        umma::mbar_arrive_expect_tx(&raw_full[slot], C::FRAME);
        umma::tma_load_4d(raw + slot * C::RAW_STRIDE, &fmap, 0, 0, 0, map.src(mf), &raw_full[slot]);
        for (int pt = 0; pt < C::NTILE; ++pt, ++it) {
          const int ts = it & 1;
          umma::mbar_wait(&d_empty[ts], ((it >> 1) & 1) ^ 1);
          const int rows = min(C::TPX, C::PIX - pt * C::TPX);        // the last tile of a frame holds 16 pixels
          umma::mbar_arrive_expect_tx(&d_full[ts], rows * 128);
          umma::bulk_g2s(dsm + ts * C::D_SLOT, da1 + ((size_t)mf * C::PIX + (size_t)pt * C::TPX) * 32, rows * 128, &d_full[ts]);
        }
      }
    }
  }
}

// partial: >= grid slabs of 257 x 32 floats; returns the number of slabs written (the grid) in *nsplit
inline int launch_conv1_wgrad_tma(cudaStream_t s, const uint8_t* frames, int nframes_total, int nframes_bwd, const RowMap& map,
                                  const float* da1, float* partial, size_t partial_floats, int* nsplit) {
  using Key = std::tuple<const uint8_t*, int>;
  static thread_local std::map<Key, CUtensorMap> cache;
  const Key key{frames, nframes_total};
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    DRL_TRY(conv1_frame_map(frames, nframes_total, &m));
    it = cache.emplace(key, m).first;
  }
  static bool attr_done = false;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(conv1_wgrad_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Conv1WgTma::SMEM_BYTES));
    attr_done = true;
  }
  const int grid = std::min(nframes_bwd, device_sm_count());
  if ((size_t)grid * Conv1WgTma::SLAB > partial_floats) { set_error("conv1_wgrad: partial buffer too small"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK((launch_k(conv1_wgrad_tma_kernel, grid, Conv1WgTma::NT, Conv1WgTma::SMEM_BYTES, s, it->second, da1, partial, map,
                           nframes_bwd)));
  *nsplit = grid;
  return DRL_OK;
}

}  // namespace drl
