// gemm_umma_persist.cuh -- persistent, warp-specialised variant of the wgmma 3xTF32 gather-GEMM
// (same operand layouts / loaders / epilogues as gemm_umma.cuh; see there for the math and the layouts).
//
//   grid = one CTA per SM; every CTA walks the tile list  tile = blockIdx.x, += gridDim.x  (m fastest)
//   warps 0..PW-1   PRODUCERS   gather -> hi/lo split -> swizzled smem stage (ring continues across tiles,
//                               register double buffering continues across tile boundaries)
//   warps PW..PW+7  CONSUMERS   two warpgroups (rows 0-63 / 64-127): wgmma into the register accumulator, hand each
//                               stage back once its MMAs are complete, then run the epilogue of the tile through
//                               their own staging tiles -- while the producers already fill the ring for the next
//                               tile
#pragma once
#include <algorithm>

#include "gemm_umma.cuh"

namespace drl {

template <int BN_, int STAGES_, int PW_ = 8>
struct UmmaPCfg {
  static constexpr int BM = 128, BN = BN_, BK = 32, STAGES = STAGES_, PW = PW_;
  static constexpr int NPROD = PW * 32;
  static constexpr int NT = NPROD + wg::kConsumerThreads;   // producers + two consumer warpgroups
  static constexpr int MINB = 1;
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN must be a power of two in [32,256]");
  static_assert(STAGES >= 2, "consumers hand a stage back only after the next stage's MMAs are issued");
  static_assert(BN / 2 + 40 <= 65536 / NT, "accumulator does not fit the register budget: fewer producer warps");
};

struct PTile {
  int tile, t, ntl, m0, n0, z, k0, k1, mt;
  bool valid;
};

template <class Cfg, class AL, class BL, class EP>
__global__ void __launch_bounds__(Cfg::NT, 1)
gemm_umma_persist_kernel(const AL al, const BL bl, const EP ep, int M, int N, int K, int kchunk, int kstep,
                         int mtiles, int ntn, int total_tiles) {
  kernel_prologue();
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, STAGES = Cfg::STAGES, NPROD = Cfg::NPROD, PW = Cfg::PW;
  constexpr bool AK = AL::kContigK, BKc = BL::kContigK;
  using SM = UmmaSmem<Cfg, AL, BL>;
  using TA = typename SM::TA;
  using TB = typename SM::TB;
  constexpr bool AEX = SM::AEX;
  constexpr bool A16 = loader_vec16<AL>::value;
  constexpr int NGA = BM * BK / 4, NGB = BN * BK / 4;
  constexpr bool BPT = loader_pretiled<BL>::value;
  constexpr int GA = (A16 ? NGA / 4 : NGA) / NPROD, GB = BPT ? 1 : NGB / NPROD;
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

  auto setup = [&](PTile& p, int tile) {
    p.tile = tile;
    p.valid = tile < total_tiles;
    if (!p.valid) return;
    p.mt = tile % mtiles;
    const int rest = tile / mtiles;
    const int nt = rest % ntn;
    p.z = rest / ntn;
    p.m0 = p.mt * BM;
    p.n0 = nt * BN;
    p.k0 = p.z * kstep;
    p.k1 = min(K, p.k0 + kchunk);
    p.ntl = (p.k1 - p.k0 + BK - 1) / BK;
    p.t = 0;
  };
  auto advance = [&](PTile& p) {
    if (++p.t >= p.ntl) setup(p, p.tile + gridDim.x);
  };

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      umma::mbar_init(&full[s], NPROD);
      umma::mbar_init(&empty[s], wg::kConsumerWGs);
    }
    umma::fence_barrier_init();
  }
  __syncthreads();

  if (warp < PW) {
    // ================= PRODUCERS =================
    // static (tile independent) part of the group assignment
    int a_r[GA], a_k[GA], a_o[GA], b_r[GB], b_k[GB], b_o[GB];
#pragma unroll
    for (int i = 0; i < GA; ++i) {
      const int g = tid + i * NPROD;
      if (A16) {
        if (AK) { a_r[i] = g % BM; a_k[i] = (g / BM) * 16; a_o[i] = a_r[i]; }
        else { a_r[i] = (g / BK) * 16; a_k[i] = g % BK; a_o[i] = a_r[i]; }
      } else if (AK) {
        a_r[i] = g >> 3; a_k[i] = (g & 7) * 4; a_o[i] = TA::chunk_off(a_r[i], a_k[i]);
      } else {
        a_r[i] = (g % (BM / 4)) * 4; a_k[i] = g / (BM / 4); a_o[i] = TA::chunk_off(a_r[i], a_k[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < GB; ++i) {
      const int g = tid + i * NPROD;
      if (BPT) { b_r[i] = 0; b_k[i] = 0; }
      else if (BKc) { b_r[i] = g >> 3; b_k[i] = (g & 7) * 4; }
      else { b_r[i] = (g % (BN / 4)) * 4; b_k[i] = g / (BN / 4); }
      b_o[i] = TB::chunk_off(b_r[i], b_k[i]);
    }
    float4 csum[GB];
#pragma unroll
    for (int i = 0; i < GB; ++i) csum[i] = zero4();

    auto gload = [&](const PTile& p, ARaw (&ra)[GA], float4 (&rb)[GB]) {
      const int kb = p.k0 + p.t * BK;
#pragma unroll
      for (int i = 0; i < GA; ++i) {
        const int m = p.m0 + a_r[i];
        const typename AL::Row row = al.row(p.z, m < M ? m : -1);
        const int k = kb + a_k[i];
        if constexpr (A16) ra[i] = (k < p.k1) ? al.load_raw16(row, k) : make_uint4(0u, 0u, 0u, 0u);
        else ra[i] = (k < p.k1) ? al.load(row, k) : zero4();
      }
      if constexpr (!BPT) {
#pragma unroll
        for (int i = 0; i < GB; ++i) {
          const int n = p.n0 + b_r[i];
          const typename BL::Row row = bl.row(p.z, n < N ? n : -1);
          const int k = kb + b_k[i];
          rb[i] = (k < p.k1) ? bl.load(row, k) : zero4();
        }
      }
    };
    auto publish = [&](const PTile& p, int q, const ARaw (&ra)[GA], const float4 (&rb)[GB]) {
      const int s = q % STAGES;
      const uint32_t ph = (q / STAGES) & 1;
      umma::mbar_wait(&empty[s], ph ^ 1);
      uint8_t* st = smem + s * SM::STAGE_BYTES;
      if constexpr (BPT) {
        if (tid == 0) {
          const int kt = (p.k0 + p.t * BK) / BK;
          umma::mbar_expect_tx(&full[s], 2 * SM::B_BYTES);
          umma::bulk_g2s(st + OFF_BHI, bl.image + ((size_t)(p.n0 / BN) * bl.ktiles + kt) * (size_t)(2 * SM::B_BYTES),
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
      const bool cs_tile = kColSum && p.mt == 0;
      if constexpr (!BPT) {
#pragma unroll
        for (int i = 0; i < GB; ++i) {
          float4 h, l;
          umma::split4(rb[i], h, l);
          TB::put(st + OFF_BHI, b_o[i], h);
          TB::put(st + OFF_BLO, b_o[i], l);
          if (cs_tile) { csum[i].x += rb[i].x; csum[i].y += rb[i].y; csum[i].z += rb[i].z; csum[i].w += rb[i].w; }
        }
      }
      umma::fence_proxy_async();
      umma::mbar_arrive(&full[s]);
      if (cs_tile && p.t == p.ntl - 1) {
        // bias-gradient row of this (n-tile, z): column sums of B over the tile's K range, fixed order
        float4 acc = zero4();
#pragma unroll
        for (int i = 0; i < GB; ++i) { acc.x += csum[i].x; acc.y += csum[i].y; acc.z += csum[i].z; acc.w += csum[i].w; csum[i] = zero4(); }
        asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory");      // previous use of the scratch is over
        cs_scratch[tid] = acc;
        asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory");
        if (tid < BN / 4) {
          float4 tot = zero4();
          for (int j = tid; j < NPROD; j += BN / 4) {
            const float4 v = cs_scratch[j];
            tot.x += v.x; tot.y += v.y; tot.z += v.z; tot.w += v.w;
          }
          const int n = p.n0 + tid * 4;
          if (n < N) ep.store_colsum(p.z, n, tot.x);
          if (n + 1 < N) ep.store_colsum(p.z, n + 1, tot.y);
          if (n + 2 < N) ep.store_colsum(p.z, n + 2, tot.z);
          if (n + 3 < N) ep.store_colsum(p.z, n + 3, tot.w);
        }
      }
    };

    PTile ld, pb;
    setup(ld, blockIdx.x);
    pb = ld;
    ARaw ra0[GA], ra1[GA];
    float4 rb0[GB], rb1[GB];
    int q = 0;
    if (ld.valid) { gload(ld, ra0, rb0); advance(ld); }
#pragma unroll 1
    while (pb.valid) {
      if (ld.valid) { gload(ld, ra1, rb1); advance(ld); }
      publish(pb, q, ra0, rb0);
      advance(pb); ++q;
      if (!pb.valid) break;
      if (ld.valid) { gload(ld, ra0, rb0); advance(ld); }
      publish(pb, q, ra1, rb1);
      advance(pb); ++q;
    }
  } else {
    // ================= CONSUMERS (warps PW .. PW+7: warpgroup cw = rows 64 cw .. 64 cw + 63) =================
    const int ct = tid - NPROD, cw = ct >> 7, cwarp = (ct >> 5) & 3;
    uint8_t* stg = aux + SM::AUX_BYTES + (ct >> 5) * wg::kEpiWarpBytes;   // dedicated staging: the stages stay live here
    PTile p;
    setup(p, blockIdx.x);
    int q = 0;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    while (p.valid) {
      const int ntl = p.ntl;
      for (int t = 0; t < ntl; ++t, ++q) {
        const int s = q % STAGES;
        umma::mbar_wait(&full[s], (q / STAGES) & 1);
        const uint32_t st = umma::smem_u32(smem + s * SM::STAGE_BYTES);
        const uint32_t a_hi = st + cw * 64 * 128;
        wg::fence_operand(acc);
        wg::fence();
        tf32_stage_mmas<BN, AEX, BK, TA, TB>(acc, a_hi, a_hi + OFF_ALO, st + OFF_BHI, st + OFF_BLO, t == 0);
        wg::commit();
        wg::wait<1>();                                 // the MMAs of the previous stage are complete: hand it back
        wg::fence_operand(acc);
        if (t > 0 && (ct & 127) == 0) umma::mbar_arrive(&empty[(q - 1) % STAGES]);
      }
      wg::wait<0>();
      wg::fence_operand(acc);
      if ((ct & 127) == 0) umma::mbar_arrive(&empty[(q - 1) % STAGES]);
      wg_epilogue<BN>(ep, acc, stg, lane, p.z, p.m0 + cw * 64 + cwarp * 16, p.n0, M, N);
      setup(p, p.tile + gridDim.x);
    }
  }
}

inline int device_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

template <class Cfg, class AL, class BL, class EP>
inline int launch_gemm_umma_persist(cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                                    int zcount, int kchunk, int kstep) {
  using SM = UmmaSmem<Cfg, AL, BL>;
  static bool attr_done = false;
  auto kern = gemm_umma_persist_kernel<Cfg, AL, BL, EP>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::BYTES + 8 * wg::kEpiWarpBytes));
    attr_done = true;
  }
  if ((AL::kContigK || BL::kContigK) && (K % 4 != 0 || kchunk % 4 != 0)) {
    set_error("gemm_umma_persist: K (%d) and kchunk (%d) must be multiples of 4 for K-contiguous operands", K, kchunk);
    return DRL_ERR_INVALID;
  }
  if (kchunk < 1 || K < 1) { set_error("gemm_umma_persist: empty K range"); return DRL_ERR_INVALID; }
  const int mtiles = cdiv(M, Cfg::BM), ntn = cdiv(N, Cfg::BN);
  const long long total = (long long)mtiles * ntn * zcount;
  if (total > 0x7fffffffLL) { set_error("gemm_umma_persist: too many tiles"); return DRL_ERR_INVALID; }
  const int grid = (int)std::min<long long>(total, device_sm_count());
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT, SM::BYTES + 8 * wg::kEpiWarpBytes, s, al, bl, ep, M, N, K, kchunk, kstep,
                           mtiles, ntn, (int)total)));
  return DRL_OK;
}

}  // namespace drl
