// policy_head.cuh -- device pieces shared by the policy engines' head kernels (policy.cu: policy_head_fused;
// apex_policy.cu: apex_policy_head): the 256 x 256 dense layer over the kHR rows of a CTA, and the sampler of numpy's
// RandomState.choice(A, p=policy).
#pragma once
#include "kernels.h"

namespace drl {

// rows per head CTA: with 8 rows per CTA a head's weights are read from L2 once per 8 rows
constexpr int kHR = 8;

// out[r][u] = relu(sum_k in[r][k] W[k][u] + b[u]) for the kHR rows of the CTA (W [256][256] row-major), 256 threads.
// Thread (q, g) owns columns 4q..4q+3 over the K quarter g, with 16 float4 weight loads in flight; the four K partials
// (part: [4][kHR][256]) are added in fixed order (0 + 1) + 2 + 3.
__device__ __forceinline__ void dense256_relu(const float* __restrict__ in, const float* __restrict__ W,
                                              const float* __restrict__ b, float* part, float* out, int tid) {
  const int q = tid & 63, g = tid >> 6;
  float acc[kHR][4];
#pragma unroll
  for (int r = 0; r < kHR; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
#pragma unroll 1
  for (int kk = 0; kk < 64; kk += 16) {
    float4 wv[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) wv[j] = ldg4(W + (size_t)(g * 64 + kk + j) * 256 + 4 * q);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int k = g * 64 + kk + j;
#pragma unroll
      for (int r = 0; r < kHR; ++r) {
        const float x = in[r * 256 + k];
        acc[r][0] = fmaf(x, wv[j].x, acc[r][0]);
        acc[r][1] = fmaf(x, wv[j].y, acc[r][1]);
        acc[r][2] = fmaf(x, wv[j].z, acc[r][2]);
        acc[r][3] = fmaf(x, wv[j].w, acc[r][3]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kHR; ++r)
    reinterpret_cast<float4*>(part + (g * kHR + r) * 256)[q] = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
  __syncthreads();
  const float bias = __ldg(b + tid);
#pragma unroll
  for (int r = 0; r < kHR; ++r) {
    const float* p = part + r * 256 + tid;
    const float v = ((p[0] + p[kHR * 256]) + p[2 * kHR * 256]) + p[3 * kHR * 256];
    out[r * 256 + tid] = fmaxf(v + bias, 0.f);
  }
  __syncthreads();
}

// The action of numpy's RandomState.choice(A, p=policy) for the uniform draw uniform[m], from one thread: cdf =
// cumsum(float64(policy)) / cdf[A-1] in index order; action = #(cdf <= u), clamped to A - 1 -- the
// searchsorted(cdf, u, side='right') of the legacy generator.  `policy` is the row's A probabilities (shared memory).
__device__ __forceinline__ int sample_choice(const float* policy, int A, const double* uniform, int m) {
  double total = 0.0;
  for (int i = 0; i < A; ++i) total += (double)policy[i];
  const double uu = uniform[m];
  double run = 0.0;
  int cnt = 0;
  for (int i = 0; i < A; ++i) {
    run += (double)policy[i];
    cnt += (run / total <= uu) ? 1 : 0;
  }
  return cnt < A - 1 ? cnt : A - 1;
}

}  // namespace drl
