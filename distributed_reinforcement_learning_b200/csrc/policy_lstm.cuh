// policy_lstm.cuh -- the skinny split-K LSTM GEMM of the policy engines: z = [a3 | table[pa] | h0] W for n <= 64 rows,
// as partial sums per K split (policy.cu: IMPALA, L = 256, N = 1024; r2d2_policy.cu: R2D2, L = 64, N = 256).  The
// learners' LSTM GEMMs are shaped for hundreds of rows; at n <= 64 the cost is streaming the fp32 weights once, over
// every SM.
#pragma once
#include "gemm_umma.cuh"   // umma:: mbarrier / bulk-copy helpers
#include "kernels.h"

namespace drl {

// grid (N / kLN column chunks) x (kSplits K splits), each CTA streaming its kK x 128 fp32 slab of W once.  The slab
// arrives by kK row-wise cp.async.bulk copies of 512 B (all in flight at once, completing on kLStages mbarriers so the
// FFMA loop starts on the first third); the CTA's [R x kK] slice of x is gathered into shared memory meanwhile.
// Thread (c, g): columns c and c + 64 for the rows [g R/4, (g+1) R/4) -- per 4 k: 8 conflict-free LDS of W and R/4
// broadcast LDS.128 of x for 2 R FFMA.
constexpr int kLN = 128;
constexpr int kLStages = 3;
constexpr int kLThreads = 256;

// L = width of the recurrent state h0 (the last L rows of W), N = 4 L gate columns, kSplits = K splits
template <int L, int kSplits>
struct LstmSplit {
  static constexpr int N = 4 * L;
  static constexpr int K = Geo::FLAT + Geo::EMB + L;
  static constexpr int kK = K / kSplits;             // rows of W per CTA
  static constexpr int kStageK = kK / kLStages;
  static_assert(kK * kSplits == K && kStageK * kLStages == kK && kStageK % 4 == 0, "LSTM split tiling");
  static_assert(Geo::FLAT % 4 == 0 && (Geo::FLAT + Geo::EMB) % 4 == 0 && kK % 4 == 0 && N % kLN == 0, "float4 gather");
  static constexpr size_t smem_bytes(int R) { return (size_t)kK * kLN * 4 + (size_t)R * kK * 4 + 8 * kLStages; }
};

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(bar)), "r"(bytes) : "memory");
}

template <int R, int L, int kSplits>
__global__ void __launch_bounds__(kLThreads, 1) policy_lstm_fwd_kernel(
    const float* __restrict__ a3, const float* __restrict__ table, const int32_t* __restrict__ pa,
    const float* __restrict__ h0, const float* __restrict__ w, float* __restrict__ zpart, int n) {
  using Sp = LstmSplit<L, kSplits>;
  constexpr int kK = Sp::kK, kStageK = Sp::kStageK, N = Sp::N;
  kernel_prologue();
  extern __shared__ __align__(128) uint8_t smem[];
  float* sw = reinterpret_cast<float*>(smem);     // [kK][kLN]
  float* sx = sw + kK * kLN;                       // [R][kK]
  uint64_t* bar = reinterpret_cast<uint64_t*>(sx + R * kK);
  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * kLN, split = blockIdx.y, k0 = split * kK;
  if (tid == 0) {
    for (int s = 0; s < kLStages; ++s) umma::mbar_init(&bar[s], 1);
    umma::fence_barrier_init();
  }
  __syncthreads();
  if (tid < 32) {
    for (int s = 0; s < kLStages; ++s) {
      if (tid == 0) mbar_arrive_expect_tx(&bar[s], kStageK * kLN * 4);
      __syncwarp();
      for (int k = s * kStageK + tid; k < (s + 1) * kStageK; k += 32)
        umma::bulk_g2s(sw + k * kLN, w + (size_t)(k0 + k) * N + n0, kLN * 4, &bar[s]);
    }
  }
  // x = [a3 | table[pa] | h0] over this CTA's K range (every float4 lies in one of the three parts); rows >= n are zero
  constexpr int K4 = kK / 4;
  for (int i = tid; i < R * K4; i += kLThreads) {
    const int r = i / K4, q = i - r * K4, k = k0 + 4 * q;
    float4 v = zero4();
    if (r < n) {
      if (k < Geo::FLAT) v = ldg4(a3 + (size_t)r * Geo::FLAT + k);
      else if (k < Geo::FLAT + Geo::EMB) v = ldg4(table + (size_t)__ldg(pa + r) * Geo::EMB + (k - Geo::FLAT));
      else v = ldg4(h0 + (size_t)r * L + (k - Geo::FLAT - Geo::EMB));
    }
    reinterpret_cast<float4*>(sx + r * kK)[q] = v;
  }
  __syncthreads();
  constexpr int RT = R / 4;
  const int c = tid & 63, r0 = (tid >> 6) * RT;
  float acc0[RT], acc1[RT];
#pragma unroll
  for (int r = 0; r < RT; ++r) acc0[r] = acc1[r] = 0.f;
  for (int s = 0; s < kLStages; ++s) {
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

// zpart [kSplits][n][4 L] for n <= 64 rows: the smallest row tile R in {8, 16, 32, 64} that holds n
template <int L, int kSplits>
int launch_policy_lstm(cudaStream_t s, const float* a3, const float* table, const int32_t* pa, const float* h0,
                       const float* w, float* zpart, int n) {
  using Sp = LstmSplit<L, kSplits>;
  const dim3 grid(Sp::N / kLN, kSplits);
  if (n <= 8)
    DRL_CUDA_CHECK((launch_k(policy_lstm_fwd_kernel<8, L, kSplits>, grid, kLThreads, Sp::smem_bytes(8), s, a3, table,
                             pa, h0, w, zpart, n)));
  else if (n <= 16)
    DRL_CUDA_CHECK((launch_k(policy_lstm_fwd_kernel<16, L, kSplits>, grid, kLThreads, Sp::smem_bytes(16), s, a3, table,
                             pa, h0, w, zpart, n)));
  else if (n <= 32)
    DRL_CUDA_CHECK((launch_k(policy_lstm_fwd_kernel<32, L, kSplits>, grid, kLThreads, Sp::smem_bytes(32), s, a3, table,
                             pa, h0, w, zpart, n)));
  else
    DRL_CUDA_CHECK((launch_k(policy_lstm_fwd_kernel<64, L, kSplits>, grid, kLThreads, Sp::smem_bytes(64), s, a3, table,
                             pa, h0, w, zpart, n)));
  return DRL_OK;
}

template <int L, int kSplits>
int set_policy_lstm_attributes() {
  using Sp = LstmSplit<L, kSplits>;
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_lstm_fwd_kernel<8, L, kSplits>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)Sp::smem_bytes(8)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_lstm_fwd_kernel<16, L, kSplits>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(16)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_lstm_fwd_kernel<32, L, kSplits>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(32)));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_lstm_fwd_kernel<64, L, kSplits>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Sp::smem_bytes(64)));
  return DRL_OK;
}

}  // namespace drl
