// gemm_simt.cuh -- generic gather-GEMM on the FP32 FFMA pipe.
//
//   C(z; m, n) = sum_{k in [k0, k1)} A(z; m, k) * B(z; k, n)
//
// A and B are produced by loader functors (im2col gathers, concatenations, transposes), C is
// consumed by an epilogue functor (bias/ReLU, ReLU-mask, split-K partials, bias-gradient column
// sums).  blockIdx.z is either a split-K index (k0 = z * kchunk) or a batch index (kstep = 0).
//
// Loader concept (AL for the M side, BL for the N side):
//   static constexpr bool kContigK;   // true : load() returns (idx, k..k+3)      ("K-major")
//                                     // false: load() returns (idx..idx+3, k)    ("M/N-major")
//   struct Row;                       // per-index context, hoisted out of the K loop
//   Row    row(int z, int idx) const; // idx < 0  => invalid row (loads return 0)
//   float4 load(const Row&, int k) const;
// Epilogue concept:
//   template<int V> void store(int z, int m, int n, const float (&v)[V]) const;  // V in {1,4}
//   static constexpr bool kColSum;  void store_colsum(int z, int n, float v) const;
//
// Tile: BM x BN x BK, thread micro-tile TM x TN (multiples of 4), NT = (BM/TM)*(BN/TN) threads,
// register-prefetch double buffering with one __syncthreads per K tile.  K ranges and all
// contiguous-dimension extents must be multiples of 4 (checked by the host launchers).
#pragma once
#include "common.cuh"

namespace drl {

template <int BM_, int BN_, int BK_, int TM_, int TN_>
struct TileCfg {
  static constexpr int BM = BM_, BN = BN_, BK = BK_, TM = TM_, TN = TN_;
  static constexpr int TX = BN / TN, TY = BM / TM, NT = TX * TY;
  static constexpr int QM = TM / 4, QN = TN / 4;
  static_assert(TM % 4 == 0 && TN % 4 == 0 && BK % 4 == 0, "micro tile must be float4 friendly");
  static_assert((BM * BK / 4) % NT == 0 && (BN * BK / 4) % NT == 0, "loader groups must divide");
};

template <class Cfg, bool AContigK, bool BContigK>
struct SmemLayout {
  // A: K-contig -> [BM][BK+4]; M-contig -> [BK][BM+4].  B: K-contig -> [BN][BK+4]; N-contig -> [BK][BN+4]
  static constexpr int SA = AContigK ? (Cfg::BK + 4) : (Cfg::BM + 4);
  static constexpr int SB = BContigK ? (Cfg::BK + 4) : (Cfg::BN + 4);
  static constexpr int A_ELEMS = AContigK ? Cfg::BM * SA : Cfg::BK * SA;
  static constexpr int B_ELEMS = BContigK ? Cfg::BN * SB : Cfg::BK * SB;
  static constexpr int BYTES = 2 * (A_ELEMS + B_ELEMS) * 4;
};

// KS > 1: in-CTA split-K for the small, latency-bound dense layers (heads): KS thread groups of Cfg::NT threads each
// own every KS-th K tile (their own shared-memory buffers, a named barrier per group), so the K tiles of one output
// tile are loaded and multiplied concurrently instead of one after the other; the partial tiles are then summed by
// group 0 in the fixed order 0..KS-1 (deterministic) before the unchanged epilogue.  KS = 1 is the original kernel.
template <class Cfg, class AL, class BL, class EP, int KS = 1>
__global__ void __launch_bounds__(Cfg::NT * KS)
gemm_simt_kernel(const AL al, const BL bl, const EP ep, int M, int N, int K, int kchunk, int kstep) {
  kernel_prologue();
  constexpr int BM = Cfg::BM, BN = Cfg::BN, BK = Cfg::BK, TM = Cfg::TM, TN = Cfg::TN;
  constexpr int NT = Cfg::NT, TX = Cfg::TX, QM = Cfg::QM, QN = Cfg::QN;
  constexpr bool AK = AL::kContigK, BKc = BL::kContigK;
  using SL = SmemLayout<Cfg, AK, BKc>;
  constexpr int SA = SL::SA, SB = SL::SB;
  constexpr int GA = BM * BK / 4 / NT, GB = BN * BK / 4 / NT;

  extern __shared__ __align__(16) float smem_all[];
  const int grp = KS > 1 ? (int)threadIdx.x / NT : 0;
  float* smem = smem_all + (size_t)grp * (2 * (SL::A_ELEMS + SL::B_ELEMS));
  float* As = smem;                       // 2 buffers
  float* Bs = smem + 2 * SL::A_ELEMS;     // 2 buffers
  auto group_sync = [&]() {
    if (KS == 1) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(NT) : "memory");
  };

  const int tid = KS > 1 ? (int)threadIdx.x % NT : (int)threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int z = blockIdx.z;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int k0 = z * kstep;
  const int k1 = min(K, k0 + kchunk);
  const int ntiles_all = (k1 - k0 + BK - 1) / BK;
  const int ntiles = KS > 1 ? (ntiles_all > grp ? (ntiles_all - grp + KS - 1) / KS : 0) : ntiles_all;   // this group's

  // ---- loader assignment: group g = tid + i*NT --------------------------------------
  // K-contig : row = g / (BK/4), kq = g % (BK/4)  -> smem [row][kq*4]
  // M-contig : kk  = g / (BM/4), mq = g % (BM/4)  -> smem [kk][mq*4]
  typename AL::Row arow[GA];
  typename BL::Row brow[GB];
  int a_k[GA], a_s[GA], b_k[GB], b_s[GB];
#pragma unroll
  for (int i = 0; i < GA; ++i) {
    const int g = tid + i * NT;
    if (AK) {
      const int r = g / (BK / 4), kq = g % (BK / 4);
      const int m = m0 + r;
      arow[i] = al.row(z, m < M ? m : -1);
      a_k[i] = kq * 4;
      a_s[i] = r * SA + kq * 4;
    } else {
      const int kk = g / (BM / 4), mq = g % (BM / 4);
      const int m = m0 + mq * 4;
      arow[i] = al.row(z, m < M ? m : -1);
      a_k[i] = kk;
      a_s[i] = kk * SA + mq * 4;
    }
  }
#pragma unroll
  for (int i = 0; i < GB; ++i) {
    const int g = tid + i * NT;
    if (BKc) {
      const int r = g / (BK / 4), kq = g % (BK / 4);
      const int n = n0 + r;
      brow[i] = bl.row(z, n < N ? n : -1);
      b_k[i] = kq * 4;
      b_s[i] = r * SB + kq * 4;
    } else {
      const int kk = g / (BN / 4), nq = g % (BN / 4);
      const int n = n0 + nq * 4;
      brow[i] = bl.row(z, n < N ? n : -1);
      b_k[i] = kk;
      b_s[i] = kk * SB + nq * 4;
    }
  }

  float4 ra[GA], rb[GB];
  auto gload = [&](int t) {
    const int kb = k0 + (grp + t * KS) * BK;
#pragma unroll
    for (int i = 0; i < GA; ++i) {
      const int k = kb + a_k[i];
      ra[i] = (k < k1) ? al.load(arow[i], k) : zero4();
    }
#pragma unroll
    for (int i = 0; i < GB; ++i) {
      const int k = kb + b_k[i];
      rb[i] = (k < k1) ? bl.load(brow[i], k) : zero4();
    }
  };
  auto sstore = [&](int buf) {
    float* a = As + buf * SL::A_ELEMS;
    float* b = Bs + buf * SL::B_ELEMS;
#pragma unroll
    for (int i = 0; i < GA; ++i) *reinterpret_cast<float4*>(a + a_s[i]) = ra[i];
#pragma unroll
    for (int i = 0; i < GB; ++i) *reinterpret_cast<float4*>(b + b_s[i]) = rb[i];
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float colsum = 0.f;   // used when EP::kColSum (thread tid < BN sums column n0+tid of B)

  if (ntiles > 0) {
    gload(0);
    sstore(0);
  }
  group_sync();

  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) gload(t + 1);
    const float* a = As + buf * SL::A_ELEMS;
    const float* b = Bs + buf * SL::B_ELEMS;

    if (EP::kColSum && !BKc) {
      if (blockIdx.x == 0 && tid < BN) {
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) colsum += b[kk * SB + tid];
      }
    }

#pragma unroll
    for (int kk = 0; kk < BK; kk += 4) {
      float av[TM][4], bv[4][TN];
      if (AK) {
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          const int ml = (i / 4) * (BM / QM) + ty * 4 + (i % 4);
          const float4 v = *reinterpret_cast<const float4*>(a + ml * SA + kk);
          av[i][0] = v.x; av[i][1] = v.y; av[i][2] = v.z; av[i][3] = v.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int q = 0; q < QM; ++q) {
            const float4 v = *reinterpret_cast<const float4*>(a + (kk + j) * SA + q * (BM / QM) + ty * 4);
            av[q * 4 + 0][j] = v.x; av[q * 4 + 1][j] = v.y; av[q * 4 + 2][j] = v.z; av[q * 4 + 3][j] = v.w;
          }
      }
      if (BKc) {
        // strided column mapping n = j*TX + tx : conflict-free float4 reads along K
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          const float4 v = *reinterpret_cast<const float4*>(b + (j * TX + tx) * SB + kk);
          bv[0][j] = v.x; bv[1][j] = v.y; bv[2][j] = v.z; bv[3][j] = v.w;
        }
      } else {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
#pragma unroll
          for (int q = 0; q < QN; ++q) {
            const float4 v = *reinterpret_cast<const float4*>(b + (kk + jj) * SB + q * (BN / QN) + tx * 4);
            bv[jj][q * 4 + 0] = v.x; bv[jj][q * 4 + 1] = v.y; bv[jj][q * 4 + 2] = v.z; bv[jj][q * 4 + 3] = v.w;
          }
      }
#pragma unroll
      for (int j4 = 0; j4 < 4; ++j4)
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i][j4], bv[j4][j], acc[i][j]);
    }

    if (t + 1 < ntiles) sstore(buf ^ 1);
    group_sync();
  }

  if (KS > 1) {
    // partial tiles of groups 1..KS-1 -> their own (now idle) buffers, float4 e of thread tid at [(e * NT + tid)]
    static_assert(KS == 1 || 2 * (SL::A_ELEMS + SL::B_ELEMS) >= NT * TM * TN + BN, "partial tile must fit the group's buffers");
    if (grp > 0) {
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; j += 4)
          *reinterpret_cast<float4*>(smem + ((i * TN + j) / 4 * NT + tid) * 4) =
              make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
      if (EP::kColSum && !BKc && tid < BN) smem[NT * TM * TN + tid] = colsum;
    }
    __syncthreads();
    if (grp > 0) return;
#pragma unroll 1
    for (int g = 1; g < KS; ++g) {
      const float* part = smem_all + (size_t)g * (2 * (SL::A_ELEMS + SL::B_ELEMS));
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
          const float4 v = *reinterpret_cast<const float4*>(part + ((i * TN + j) / 4 * NT + tid) * 4);
          acc[i][j] += v.x; acc[i][j + 1] += v.y; acc[i][j + 2] += v.z; acc[i][j + 3] += v.w;
        }
      if (EP::kColSum && !BKc && tid < BN) colsum += part[NT * TM * TN + tid];
    }
  }

  // ---- epilogue ---------------------------------------------------------------------
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + (i / 4) * (BM / QM) + ty * 4 + (i % 4);
    if (m >= M) continue;
    if (BKc) {
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = n0 + j * TX + tx;
        if (n < N) {
          const float v[1] = {acc[i][j]};
          ep.template store<1>(z, m, n, v);
        }
      }
    } else {
#pragma unroll
      for (int q = 0; q < QN; ++q) {
        const int n = n0 + q * (BN / QN) + tx * 4;
        if (n + 3 < N) {
          const float v[4] = {acc[i][q * 4 + 0], acc[i][q * 4 + 1], acc[i][q * 4 + 2], acc[i][q * 4 + 3]};
          ep.template store<4>(z, m, n, v);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (n + j < N) {
              const float v[1] = {acc[i][q * 4 + j]};
              ep.template store<1>(z, m, n + j, v);
            }
        }
      }
    }
  }
  if (EP::kColSum && !BKc) {
    if (blockIdx.x == 0 && tid < BN && n0 + tid < N) ep.store_colsum(z, n0 + tid, colsum);
  }
}

template <class Cfg, int KS = 1, class AL, class BL, class EP>
inline int launch_gemm_simt(cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                            int zcount, int kchunk, int kstep) {
  using SL = SmemLayout<Cfg, AL::kContigK, BL::kContigK>;
  static_assert(SL::BYTES * KS <= 227 * 1024 && Cfg::NT * KS <= 1024, "in-CTA split-K does not fit");
  static bool attr_done = false;   // per instantiation
  auto kern = gemm_simt_kernel<Cfg, AL, BL, EP, KS>;
  if (!attr_done) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SL::BYTES * KS));
    attr_done = true;
  }
  if ((AL::kContigK || BL::kContigK) && (K % 4 != 0 || kchunk % 4 != 0)) {
    set_error("gemm_simt: K (%d) and kchunk (%d) must be multiples of 4 for K-contiguous operands", K, kchunk);
    return DRL_ERR_INVALID;
  }
  dim3 grid(cdiv(M, Cfg::BM), cdiv(N, Cfg::BN), zcount);
  DRL_CUDA_CHECK((launch_k(kern, grid, Cfg::NT * KS, SL::BYTES * KS, s, al, bl, ep, M, N, K, kchunk, kstep)));
  return DRL_OK;
}

// Tile configurations used by the layers.
using CfgBig = TileCfg<128, 64, 16, 8, 8>;    // 128 threads, 64 accumulators
using CfgN32 = TileCfg<128, 32, 16, 8, 4>;    // N = 32 outputs (conv1, conv2-dgrad)
using CfgMid = TileCfg<64, 64, 16, 8, 4>;     // 128 threads, small-M GEMMs (LSTM, dgrads)
using CfgSmall = TileCfg<32, 64, 64, 4, 4>;   // 128 threads, tiny dense layers: latency-bound, so few deep K tiles
using CfgWg1 = TileCfg<256, 32, 16, 8, 8>;    // conv1 wgrad: C is [256(+1) x 32]

}  // namespace drl
