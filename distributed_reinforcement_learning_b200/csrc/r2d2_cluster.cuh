// r2d2_cluster.cuh -- the R2D2 LSTM recurrence at lstm_size 256 and 512 (r2d2.cu keeps r2d2_lstm_fwd_kernel /
// r2d2_lstm_bwd_kernel for 64): the same contracts, with W_h (L x 4L fp32: 1 MB at 256, 4 MB at 512) spread over a
// thread-block cluster of CL = L / 32 CTAs (8, portable; 16, non-portable) so that it stays on chip for all S steps.
// The IMPALA learner's recurrent mode (layers.cu) runs the same bodies at 256 in their RESTART variant.
//
// CTA `rank` of a cluster owns hidden units [32 rank, 32 rank + 32) and their four gate columns (i, j, f, o): 128 local
// columns c, global column (c / 32) L + 32 rank + c % 32, so the cell update of a unit never leaves its CTA.  It holds
// W_h[:, those columns] (L x 128: 128 KB at 256, 256 KB at 512) for the whole launch: each thread 128 weights, some in
// registers and the rest in shared memory (all of them in registers at 256; at 512, where 256 KB is more than one SM's
// 227 KB of shared memory, 56 of them in the forward and 32 in BPTT).  A cluster walks R sequences at a time (8 at 256,
// 4 at 512) through the S steps as one [R x L] x [L x 128] product per CTA and step; clusters split the sequences in
// chunks of R.
//
// Forward step t: every CTA reads h_{t-1} of all L units from its own shared memory, forms its 128 gate columns, and
// each cell thread publishes its unit's masked h_t to the h buffer of every CTA of the cluster (distributed shared
// memory, double-buffered by step parity); one cluster barrier orders the steps.
// BPTT step t: each CTA forms dz of its 128 columns, then the partial dh_in[k] = sum over its columns dz W_h[k, :] for
// all L units k, and sends the 32 partials of each unit group to the CTA that owns it; the owner adds the CL partials in
// rank order at the next step.  Every sum runs in a fixed order, without atomics: the results are bit-reproducible.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace drl {

template <int L>
struct R2Clu {
  static constexpr int CL = L / 32;                 // CTAs per cluster (one per 32 hidden units)
  static constexpr int G = 4 * L;                   // gate columns of W_h
  static constexpr int NC = 128;                    // gate columns of one CTA
  static constexpr int KSEG = 128;                  // weights per thread
  static constexpr int KS = L / KSEG;               // forward: K segments of one column (2 or 4)
  static constexpr int T = NC * KS;                 // threads (= L: BPTT thread k owns row k of the slice)
  static constexpr int R = L == 256 ? 8 : 4;        // sequences per cluster pass
  // weights per thread in registers (forward, BPTT); the others in shared memory.  At 512 threads a thread has 128
  // registers: these are the largest counts that compile without spills.
  static constexpr int WREG = L == 256 ? 128 : 56, WREGB = L == 256 ? 128 : 32;
  static constexpr int WSM = KSEG - WREG, WSMB = KSEG - WREGB;
  static constexpr int E = R * NC / T;              // forward gate entries per thread
  static constexpr size_t kFwdSmem = sizeof(float) * ((size_t)KS * WSM * NC + 2 * R * L + KS * R * NC + R * NC);
  static constexpr size_t kBwdSmem = sizeof(float) * ((size_t)WSMB * L + R * NC + 2 * CL * R * 32);
  static_assert(R * 32 <= T, "one cell thread per (sequence, unit)");
  static_assert(WREG % 4 == 0 && WREGB % 4 == 0, "float4 steps");
  static_assert(kFwdSmem <= 227 * 1024 && kBwdSmem <= 227 * 1024, "shared memory of one SM");
  __device__ static __forceinline__ int gcol(int rank, int c) { return (c >> 5) * L + rank * 32 + (c & 31); }
};

// Forward: as r2d2_lstm_fwd_kernel (zx [M, 4L] already holds the split-K sum; rows m = t B + b).  Grid: a multiple of
// CL CTAs of T threads, cluster (CL, 1, 1), R2Clu<L>::kFwdSmem bytes of dynamic shared memory.
// RESTART = false (R2D2): h0 / c0 are [B, L], and done (optional, [B, S]) zeroes the state entering step t + 1.
// RESTART = true (the IMPALA learner's recurrent mode): h0 / c0 are the states the actor recorded for every step, [B, S, L]
// batch-major, and done [B, S] is required: after done[b, t] step t + 1 starts from the recorded (h0, c0)[b, t + 1]
// instead of (h_t, c_t); nothing is zeroed.
template <int L, bool RESTART>
__device__ __forceinline__ void lstm_fwd_cluster_body(
    const float* __restrict__ zx, const float* __restrict__ bias, const float* __restrict__ Wh,
    const float* __restrict__ h0, const float* __restrict__ c0, const uint8_t* __restrict__ done,
    float* __restrict__ gates, float* __restrict__ tc, float* __restrict__ hout, float* __restrict__ hin,
    float* __restrict__ cin, float* __restrict__ c_last, int B, int S) {
  using K = R2Clu<L>;
  constexpr int NC = K::NC, R = K::R, T = K::T, G = K::G;
  kernel_prologue();
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) float smem[];
  float* sW = smem;                                 // [KS][WSM / 4][NC][4]
  float* hbuf = sW + K::KS * K::WSM * NC;           // [2][R][L]: h entering the step, all L units
  float* part = hbuf + 2 * R * L;                   // [KS][R][NC]
  float* sact = part + K::KS * R * NC;              // [R][NC] activated gates
  const int tid = threadIdx.x;
  const int c = tid % NC, ks = tid / NC;
  const int gc = K::gcol(rank, c);
  float w[K::WREG];
#pragma unroll
  for (int kk = 0; kk < K::WREG; ++kk) w[kk] = __ldg(Wh + (size_t)(ks * K::KSEG + kk) * G + gc);
  for (int kk = 0; kk < K::WSM; ++kk)
    sW[((ks * (K::WSM / 4) + kk / 4) * NC + c) * 4 + (kk & 3)] = __ldg(Wh + (size_t)(ks * K::KSEG + K::WREG + kk) * G + gc);
  const bool cell = tid < R * 32;
  const int cr = tid >> 5, cu = rank * 32 + (tid & 31);   // the cell thread's sequence (in the pass) and unit
  const int nchunks = (B + R - 1) / R;
  const int cid = blockIdx.x / K::CL, ncl = gridDim.x / K::CL;
  cluster.sync();                                   // every peer runs before the first distributed store
  for (int ch = cid; ch < nchunks; ch += ncl) {
    const int b0 = ch * R;
    for (int i = tid; i < R * L; i += T) {
      const int b = b0 + i / L;
      hbuf[i] = b < B ? h0[(RESTART ? (size_t)b * S : (size_t)b) * L + i % L] : 0.f;
    }
    float c_reg = 0.f;
    if (cell && b0 + cr < B) c_reg = c0[(RESTART ? (size_t)(b0 + cr) * S : (size_t)(b0 + cr)) * L + cu];
    __syncthreads();
    for (int t = 0; t < S; ++t) {
      const float* hb = hbuf + (t & 1) * R * L;
      // the step input and done flag do not depend on the recurrence: issued before the product hides their latency
      float zin[K::E];
#pragma unroll
      for (int i = 0; i < K::E; ++i) {
        const int e = tid + i * T, b = b0 + e / NC, g = K::gcol(rank, e % NC);
        zin[i] = b < B ? bias[g] + zx[((size_t)t * B + b) * G + g] : 0.f;
      }
      const bool live = cell && b0 + cr < B;
      const float keep = (!RESTART && live && done && done[(size_t)(b0 + cr) * S + t]) ? 0.f : 1.f;
      // RESTART: step t + 1 starts from the recorded (h_rec, c_rec); read here, before the product, like zin
      bool restart = false;
      float h_rec = 0.f, c_rec = 0.f;
      if constexpr (RESTART) {
        if (live && t + 1 < S && done[(size_t)(b0 + cr) * S + t]) {
          restart = true;
          const size_t r = ((size_t)(b0 + cr) * S + t + 1) * L + cu;
          h_rec = h0[r];
          c_rec = c0[r];
        }
      }
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
      const float* hk = hb + ks * K::KSEG;
#pragma unroll
      for (int kk = 0; kk < K::WREG; kk += 4) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 h4 = *reinterpret_cast<const float4*>(hk + r * L + kk);   // broadcast
          acc[r] = fmaf(h4.x, w[kk], acc[r]);
          acc[r] = fmaf(h4.y, w[kk + 1], acc[r]);
          acc[r] = fmaf(h4.z, w[kk + 2], acc[r]);
          acc[r] = fmaf(h4.w, w[kk + 3], acc[r]);
        }
      }
#pragma unroll 4
      for (int kq = 0; kq < K::WSM / 4; ++kq) {
        const float4 w4 = *reinterpret_cast<const float4*>(sW + ((ks * (K::WSM / 4) + kq) * NC + c) * 4);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 h4 = *reinterpret_cast<const float4*>(hk + r * L + K::WREG + kq * 4);
          acc[r] = fmaf(h4.x, w4.x, acc[r]);
          acc[r] = fmaf(h4.y, w4.y, acc[r]);
          acc[r] = fmaf(h4.z, w4.z, acc[r]);
          acc[r] = fmaf(h4.w, w4.w, acc[r]);
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) part[(ks * R + r) * NC + c] = acc[r];
      __syncthreads();
#pragma unroll
      for (int i = 0; i < K::E; ++i) {
        const int e = tid + i * T, r = e / NC, cc = e % NC, b = b0 + r;
        float dot = part[r * NC + cc];
#pragma unroll
        for (int s = 1; s < K::KS; ++s) dot += part[(s * R + r) * NC + cc];
        const float pre = zin[i] + dot;
        const int gate = cc >> 5;
        const float actv = (gate == 1) ? tanhf(pre) : sigmoidf_acc(gate == 2 ? pre + 1.0f : pre);
        sact[e] = actv;
        if (b < B) gates[((size_t)t * B + b) * G + K::gcol(rank, cc)] = actv;
      }
      __syncthreads();
      if (cell) {
        const float* a = sact + cr * NC + (tid & 31);
        const float si = a[0], tj = a[32], sf = a[64], so = a[96];
        const float cv = sf * c_reg + si * tj;
        const float tcv = tanhf(cv);
        const float h = so * tcv;
        if (live) {
          const size_t o = ((size_t)t * B + b0 + cr) * L + cu;
          hin[o] = hb[cr * L + cu];
          cin[o] = c_reg;
          tc[o] = tcv;
          hout[o] = h;
          if (c_last) c_last[o] = cv;
        }
        c_reg = RESTART ? (restart ? c_rec : cv) : cv * keep;
        if (t + 1 < S) {
          float* dst = hbuf + ((t + 1) & 1) * R * L + cr * L + cu;
          const float hk2 = RESTART ? (restart ? h_rec : h) : h * keep;
#pragma unroll
          for (int q = 0; q < K::CL; ++q) *cluster.map_shared_rank(dst, q) = hk2;
        }
      }
      cluster.sync();
    }
  }
}

template <int L>
__global__ void __launch_bounds__(R2Clu<L>::T, 1) r2d2_lstm_fwd_cluster_kernel(
    const float* __restrict__ zx, const float* __restrict__ bias, const float* __restrict__ Wh,
    const float* __restrict__ h0, const float* __restrict__ c0, const uint8_t* __restrict__ done,
    float* __restrict__ gates, float* __restrict__ tc, float* __restrict__ hout, float* __restrict__ hin,
    float* __restrict__ cin, float* __restrict__ c_last, int B, int S) {
  lstm_fwd_cluster_body<L, false>(zx, bias, Wh, h0, c0, done, gates, tc, hout, hin, cin, c_last, B, S);
}

// BPTT: as r2d2_lstm_bwd_kernel (dhout, gates, tc, cin, done -> dz [M, 4L]) over S steps; done is [B, dstride].  Thread
// k (< L) holds row k of the CTA's slice, W_h[k, its 128 columns].  Grid and cluster as the forward, R2Clu<L>::kBwdSmem
// bytes of dynamic shared memory.  A done step carries nothing back from the next one, whether the forward zeroed the
// state after it (R2D2) or restarted from a recorded one (RESTART).  RESTART: dL/dh_out is the sum of two partials,
// dhout[m] + dhout[dh_stride + m] (the IMPALA actor and critic heads), added in that order.
template <int L, bool RESTART>
__device__ __forceinline__ void lstm_bwd_cluster_body(
    const float* __restrict__ dhout, size_t dh_stride, const float* __restrict__ gates, const float* __restrict__ tc,
    const float* __restrict__ cin, const float* __restrict__ Wh, const uint8_t* __restrict__ done,
    float* __restrict__ dz, int B, int S, int dstride) {
  using K = R2Clu<L>;
  constexpr int NC = K::NC, R = K::R, G = K::G, CL = K::CL;
  kernel_prologue();
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) float smem[];
  float* sW = smem;                                 // [WSM / 4][L][4]
  float* sdz = sW + K::WSMB * L;                     // [R][NC]
  float* recv = sdz + R * NC;                       // [2][CL][R][32]: partial dh_in of the owned units, per sender
  const int k = threadIdx.x;
  float w[K::WREGB];
#pragma unroll
  for (int c = 0; c < K::WREGB; ++c) w[c] = __ldg(Wh + (size_t)k * G + K::gcol(rank, c));
  for (int c = 0; c < K::WSMB; ++c)
    sW[((c / 4) * L + k) * 4 + (c & 3)] = __ldg(Wh + (size_t)k * G + K::gcol(rank, K::WREGB + c));
  const bool cell = k < R * 32;
  const int cr = k >> 5, u = k & 31, cu = rank * 32 + u;
  const int owner = k >> 5;                         // the CTA that owns unit k
  const int nchunks = (B + R - 1) / R;
  const int cid = blockIdx.x / CL, ncl = gridDim.x / CL;
  cluster.sync();
  for (int ch = cid; ch < nchunks; ch += ncl) {
    const int b = ch * R + cr;
    const bool live = cell && b < B;
    float dc_carry = 0.f;
    for (int t = S - 1; t >= 0; --t) {
      if (cell) {
        float dho = 0.f, si = 0.f, tj = 0.f, sf = 0.f, so = 0.f, tcv = 0.f, cprev = 0.f, keep = 0.f;
        size_t m = 0;
        if (live) {
          m = (size_t)t * B + b;
          const float* g = gates + m * G + cu;
          dho = dhout[m * L + cu];
          if constexpr (RESTART) dho += dhout[dh_stride + m * L + cu];
          si = g[0]; tj = g[L]; sf = g[2 * L]; so = g[3 * L];
          tcv = tc[m * L + cu];
          cprev = cin[m * L + cu];
          keep = done[(size_t)b * dstride + t] ? 0.f : 1.f;
        }
        float dh_next = 0.f;
        if (t + 1 < S) {
          const float* rv = recv + ((t + 1) & 1) * CL * R * 32 + cr * 32 + u;
#pragma unroll
          for (int q = 0; q < CL; ++q) dh_next += rv[q * R * 32];
        }
        const float dh = dho + keep * dh_next;
        const float d_o = dh * tcv * so * (1.f - so);
        const float dc = keep * dc_carry + dh * so * (1.f - tcv * tcv);
        const float di = dc * tj * si * (1.f - si);
        const float dj = dc * si * (1.f - tj * tj);
        const float df = dc * cprev * sf * (1.f - sf);
        dc_carry = dc * sf;
        float* sd = sdz + cr * NC + u;
        sd[0] = di; sd[32] = dj; sd[64] = df; sd[96] = d_o;
        if (live) {
          float* o = dz + m * G + cu;
          o[0] = di; o[L] = dj; o[2 * L] = df; o[3 * L] = d_o;
        }
      }
      __syncthreads();
      if (t > 0) {                                  // dh_in of step 0 leaves the sequence: not needed
        float acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0.f;
#pragma unroll
        for (int c = 0; c < K::WREGB; c += 4) {
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const float4 d4 = *reinterpret_cast<const float4*>(sdz + r * NC + c);   // broadcast
            acc[r] = fmaf(d4.x, w[c], acc[r]);
            acc[r] = fmaf(d4.y, w[c + 1], acc[r]);
            acc[r] = fmaf(d4.z, w[c + 2], acc[r]);
            acc[r] = fmaf(d4.w, w[c + 3], acc[r]);
          }
        }
#pragma unroll 4
        for (int cq = 0; cq < K::WSMB / 4; ++cq) {
          const float4 w4 = *reinterpret_cast<const float4*>(sW + (cq * L + k) * 4);
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const float4 d4 = *reinterpret_cast<const float4*>(sdz + r * NC + K::WREGB + cq * 4);
            acc[r] = fmaf(d4.x, w4.x, acc[r]);
            acc[r] = fmaf(d4.y, w4.y, acc[r]);
            acc[r] = fmaf(d4.z, w4.z, acc[r]);
            acc[r] = fmaf(d4.w, w4.w, acc[r]);
          }
        }
        float* dst = cluster.map_shared_rank(recv + (t & 1) * CL * R * 32 + rank * R * 32 + (k & 31), owner);
#pragma unroll
        for (int r = 0; r < R; ++r) dst[r * 32] = acc[r];
      }
      cluster.sync();
    }
  }
}

template <int L>
__global__ void __launch_bounds__(R2Clu<L>::T, 1) r2d2_lstm_bwd_cluster_kernel(
    const float* __restrict__ dhout, const float* __restrict__ gates, const float* __restrict__ tc,
    const float* __restrict__ cin, const float* __restrict__ Wh, const uint8_t* __restrict__ done,
    float* __restrict__ dz, int B, int S) {
  lstm_bwd_cluster_body<L, false>(dhout, 0, gates, tc, cin, Wh, done, dz, B, S, S);
}

// cudaLaunchKernelEx with a (cl, 1, 1) cluster: capturable into a CUDA graph like launch_k
template <class... KA, class... A>
inline cudaError_t launch_cluster_k(void (*kern)(KA...), int cl, dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                    A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cl;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KA>(args)...);
}

// Create-time set-up of a forward / BPTT kernel pair at width L (outside any capture): the dynamic shared memory and, at
// CL = 16, the non-portable cluster size; then how many clusters of the planned shape the device places at once (0:
// none -> the caller fails the create rather than let a step wait forever).
template <int L, class KF, class KB>
int lstm_cluster_setup(KF kf, KB kb, int* max_fwd, int* max_bwd) {
  using K = R2Clu<L>;
  DRL_CUDA_CHECK(cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K::kFwdSmem));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(kb, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K::kBwdSmem));
  if (K::CL > 8) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kf, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    DRL_CUDA_CHECK(cudaFuncSetAttribute(kb, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  }
  auto query = [](const void* kern, size_t smem, int* out) -> cudaError_t {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(K::CL);
    cfg.blockDim = dim3(K::T);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = K::CL;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaOccupancyMaxActiveClusters(out, kern, &cfg);
  };
  DRL_CUDA_CHECK(query((const void*)kf, K::kFwdSmem, max_fwd));
  DRL_CUDA_CHECK(query((const void*)kb, K::kBwdSmem, max_bwd));
  if (*max_fwd < 1 || *max_bwd < 1) {
    set_error("lstm_size %d: the device cannot place one cluster of %d CTAs of the recurrence kernels (forward %d, "
              "backward %d clusters)", L, K::CL, *max_fwd, *max_bwd);
    return DRL_ERR_CUDA;
  }
  return DRL_OK;
}

template <int L>
int r2d2_cluster_setup(int* max_fwd, int* max_bwd) {
  return lstm_cluster_setup<L>(r2d2_lstm_fwd_cluster_kernel<L>, r2d2_lstm_bwd_cluster_kernel<L>, max_fwd, max_bwd);
}

}  // namespace drl
