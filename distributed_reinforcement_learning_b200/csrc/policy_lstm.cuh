// policy_lstm.cuh -- the skinny split-K FP32-FFMA GEMM of the policy engines: z = [a3 | table[pa] | tail] W for n <= 64
// rows, as partial sums per K split.  As the LSTM input GEMM (tail = h0, N = 4 L gate columns, one row-major W):
// policy.cu (IMPALA, L = 256, N = 1024) and r2d2_policy.cu (R2D2, L = 64, N = 256).  As the first dense layer of the
// dueling / actor-critic heads (no tail, K = 3392): apex_policy.cu (Ape-X, N = 512 over the two [3392, 256] stream
// weights; A3C, N = 256 over the actor stream's).  The learners' GEMMs are shaped for hundreds of rows; at n <= 64 the
// cost is streaming the fp32 weights once, over every SM.
#pragma once
#include "gemm_umma.cuh"   // umma:: mbarrier / bulk-copy helpers
#include "kernels.h"

namespace drl {

// grid (N / kLN column chunks) x (kSplits K splits), each CTA streaming its kK x 128 fp32 slab of W once.  The slab
// arrives by kK row-wise cp.async.bulk copies of 512 B (all in flight at once, completing on kStages mbarriers so the
// FFMA loop starts on the first stage); the CTA's [R x kK] slice of x is gathered into shared memory meanwhile.
// Thread (c, g): columns c and c + 64 for the rows [g R/4, (g+1) R/4) -- per 4 k: 8 conflict-free LDS of W and R/4
// broadcast LDS.128 of x for 2 R FFMA.
constexpr int kLN = 128;
constexpr int kLStages = 3;
constexpr int kLThreads = 256;

// kTail = width of the tail of x (the last kTail rows of W; 0: none), kN = output columns, kSplits = K splits,
// kStages = mbarrier stages per slab, kWCols = columns per weight tensor: W is kN / kWCols row-major [K, kWCols]
// tensors side by side (w for columns [0, kWCols), w2 for the next kWCols).
template <int kTail, int kN, int kSplits, int kStages = kLStages, int kWCols = kN>
struct SkinnySplit {
  static constexpr int N = kN;
  static constexpr int K = Geo::FLAT + Geo::EMB + kTail;
  static constexpr int kK = K / kSplits;             // rows of W per CTA
  static constexpr int kStageK = kK / kStages;
  static_assert(kK * kSplits == K && kStageK * kStages == kK && kStageK % 4 == 0, "split tiling");
  static_assert(Geo::FLAT % 4 == 0 && (Geo::FLAT + Geo::EMB) % 4 == 0 && kK % 4 == 0 && N % kLN == 0, "float4 gather");
  static_assert(kN % kWCols == 0 && kN / kWCols <= 2 && kWCols % kLN == 0, "one or two weight tensors");
  static constexpr size_t smem_bytes(int R) { return (size_t)kK * kLN * 4 + (size_t)R * kK * 4 + 8 * kStages; }
};

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(bar)), "r"(bytes) : "memory");
}

template <int R, int kTail, int kN, int kSplits, int kStages, int kWCols>
__global__ void __launch_bounds__(kLThreads, 1) skinny_splitk_fwd_kernel(
    const float* __restrict__ a3, const float* __restrict__ table, const int32_t* __restrict__ pa,
    const float* __restrict__ tail, const float* __restrict__ w, float* __restrict__ zpart, int n,
    const float* __restrict__ w2) {
  using Sp = SkinnySplit<kTail, kN, kSplits, kStages, kWCols>;
  constexpr int kK = Sp::kK, kStageK = Sp::kStageK, N = Sp::N;
  kernel_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  float* sw = reinterpret_cast<float*>(smem);     // [kK][kLN]
  float* sx = sw + kK * kLN;                       // [R][kK]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sx + R * kK);
  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * kLN, split = blockIdx.y, k0 = split * kK;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) umma::mbar_init(&bar[s], 1);
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (tid < 32) {
    // with two weight tensors: the block of w / w2 (row stride kWCols) this CTA's columns lie in
    const float* wb = (kWCols == kN) ? w : (n0 < kWCols ? w + n0 : w2 + (n0 - kWCols)) + (size_t)k0 * kWCols;
    for (int s = 0; s < kStages; ++s) {
      if (tid == 0) mbar_arrive_expect_tx(&bar[s], kStageK * kLN * 4);
      __syncwarp();
      for (int k = s * kStageK + tid; k < (s + 1) * kStageK; k += 32) {
        if constexpr (kWCols == kN) umma::bulk_g2s(sw + k * kLN, w + (size_t)(k0 + k) * N + n0, kLN * 4, &bar[s]);
        else umma::bulk_g2s(sw + k * kLN, wb + (size_t)k * kWCols, kLN * 4, &bar[s]);
      }
    }
  }
  // x = [a3 | table[pa] | tail] over this CTA's K range (every float4 lies in one of the parts); rows >= n are zero
  constexpr int K4 = kK / 4;
  for (int i = tid; i < R * K4; i += kLThreads) {
    const int r = i / K4, q = i - r * K4, k = k0 + 4 * q;
    float4 v = zero4();
    if (r < n) {
      if (k < Geo::FLAT) v = ldg4(a3 + (size_t)r * Geo::FLAT + k);
      else if (kTail == 0 || k < Geo::FLAT + Geo::EMB) v = ldg4(table + (size_t)__ldg(pa + r) * Geo::EMB + (k - Geo::FLAT));
      else v = ldg4(tail + (size_t)r * kTail + (k - Geo::FLAT - Geo::EMB));
    }
    reinterpret_cast<float4*>(sx + r * kK)[q] = v;
  }
  __syncthreads();
  constexpr int RT = R / 4;
  const int c = tid & 63, r0 = (tid >> 6) * RT;
  float acc0[RT], acc1[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) acc0[r] = acc1[r] = 0.f;
  for (int s = 0; s < kStages; ++s) {
    umma::mbar_wait(&bar[s], 0);
#pragma unroll 2
    for (int k = s * kStageK; k < (s + 1) * kStageK; k += 4) {
      float w0[4], w1[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        w0[j] = sw[(k + j) * kLN + c];
        w1[j] = sw[(k + j) * kLN + c + 64];
      }
#pragma unroll
      for (int r = 0; r < RT; ++r) {
        const float4 x = *reinterpret_cast<const float4*>(sx + (r0 + r) * kK + k);
        acc0[r] = fmaf(x.x, w0[0], acc0[r]);
        acc1[r] = fmaf(x.x, w1[0], acc1[r]);
        acc0[r] = fmaf(x.y, w0[1], acc0[r]);
        acc1[r] = fmaf(x.y, w1[1], acc1[r]);
        acc0[r] = fmaf(x.z, w0[2], acc0[r]);
        acc1[r] = fmaf(x.z, w1[2], acc1[r]);
        acc0[r] = fmaf(x.w, w0[3], acc0[r]);
        acc1[r] = fmaf(x.w, w1[3], acc1[r]);
      }
    }
  }
  float* out = zpart + (size_t)split * n * N + n0;
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    if (r0 + r < n) {
      out[(size_t)(r0 + r) * N + c] = acc0[r];
      out[(size_t)(r0 + r) * N + c + 64] = acc1[r];
    }
  }
}

// zpart [kSplits][n][kN] for n <= 64 rows: the smallest row tile R in {8, 16, 32, 64} that holds n
template <int kTail, int kN, int kSplits, int kStages = kLStages, int kWCols = kN>
int launch_skinny_splitk(cudaStream_t s, const float* a3, const float* table, const int32_t* pa, const float* tail,
                         const float* w, const float* w2, float* zpart, int n) {
  using Sp = SkinnySplit<kTail, kN, kSplits, kStages, kWCols>;
  const dim3 grid(Sp::N / kLN, kSplits);
  if (n <= 8)
    DRL_CUDA_CHECK((launch_k(skinny_splitk_fwd_kernel<8, kTail, kN, kSplits, kStages, kWCols>, grid, kLThreads,
                             Sp::smem_bytes(8), s, a3, table, pa, tail, w, zpart, n, w2)));
  else if (n <= 16)
    DRL_CUDA_CHECK((launch_k(skinny_splitk_fwd_kernel<16, kTail, kN, kSplits, kStages, kWCols>, grid, kLThreads,
                             Sp::smem_bytes(16), s, a3, table, pa, tail, w, zpart, n, w2)));
  else if (n <= 32)
    DRL_CUDA_CHECK((launch_k(skinny_splitk_fwd_kernel<32, kTail, kN, kSplits, kStages, kWCols>, grid, kLThreads,
                             Sp::smem_bytes(32), s, a3, table, pa, tail, w, zpart, n, w2)));
  else
    DRL_CUDA_CHECK((launch_k(skinny_splitk_fwd_kernel<64, kTail, kN, kSplits, kStages, kWCols>, grid, kLThreads,
                             Sp::smem_bytes(64), s, a3, table, pa, tail, w, zpart, n, w2)));
  return DRL_OK;
}

template <int kTail, int kN, int kSplits, int kStages = kLStages, int kWCols = kN>
int set_skinny_splitk_attributes() {
  using Sp = SkinnySplit<kTail, kN, kSplits, kStages, kWCols>;
  DRL_CUDA_CHECK(cudaFuncSetAttribute(skinny_splitk_fwd_kernel<8, kTail, kN, kSplits, kStages, kWCols>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(8)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(skinny_splitk_fwd_kernel<16, kTail, kN, kSplits, kStages, kWCols>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(16)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(skinny_splitk_fwd_kernel<32, kTail, kN, kSplits, kStages, kWCols>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(32)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(skinny_splitk_fwd_kernel<64, kTail, kN, kSplits, kStages, kWCols>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(64)));
  return DRL_OK;
}

// the LSTM input GEMM: zpart [kSplits][n][4 L], x = [a3 | table[pa] | h0], one row-major W [K, 4 L]
template <int L, int kSplits>
int launch_policy_lstm(cudaStream_t s, const float* a3, const float* table, const int32_t* pa, const float* h0,
                       const float* w, float* zpart, int n) {
  return launch_skinny_splitk<L, 4 * L, kSplits>(s, a3, table, pa, h0, w, nullptr, zpart, n);
}

template <int L, int kSplits>
int set_policy_lstm_attributes() {
  return set_skinny_splitk_attributes<L, 4 * L, kSplits>();
}

}  // namespace drl
