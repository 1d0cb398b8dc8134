// vtrace.cu -- V-trace targets/advantages (optimizer/vtrace.py:29-103) as CUDA kernels.
//
//  * vtrace_losses_kernel: the learner's fused kernel.  One warp per trajectory, lane = time step.
//    Computes both V-trace windows of agent/impala.py:68-76 (steps 0..T-3 bootstrapped by V_{T-2},
//    steps 1..T-2 bootstrapped by V_{T-1}), pg_advantage (:78-80), the three loss sums
//    (optimizer/vtrace.py:105-126) and dL/dlogits, dL/dV (SURVEY.md App. A.5) in one pass.
//    The reverse recurrence acc_t = delta_t + gamma_t c_t acc_{t+1} (optimizer/vtrace.py:88-100) is an
//    affine map composition, evaluated as a warp-shuffle suffix scan (5 shuffle rounds).
//  * vtrace_from_softmax_kernel / vtrace_fiw_kernel: the stand-alone functions with the reference's
//    signatures and layouts ([B,T,A] batch-major and [T,B] time-major).
#include <algorithm>
#include <vector>

#include "kernels.h"

namespace drl {

// suffix scan of affine maps x -> b + a*x over the lanes of a warp (lane 31 is the last element)
__device__ __forceinline__ void warp_affine_suffix_scan(float& a, float& b, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float a2 = __shfl_down_sync(0xffffffffu, a, d);
    const float b2 = __shfl_down_sync(0xffffffffu, b, d);
    if (lane + d < 32) {
      b = fmaf(a, b2, b);
      a = a * a2;
    }
  }
}

__device__ __forceinline__ float clip_reward(float r, int mode) {
  if (mode == DRL_REWARD_ABS_ONE) return fminf(fmaxf(r, -1.0f), 1.0f);       // agent/impala.py:45-46
  const float sq = tanhf(r / 5.0f);                                           // agent/impala.py:47-49
  return ((r < 0.f) ? 0.3f * sq : sq) * 5.0f;
}

// One trajectory b, one warp, lane = time step: both V-trace windows, pg_advantage, the three loss terms of this
// trajectory's steps and dL/dlogits, dL/dV.  policy / value are addressed as base + t * stride so that the same code
// reads them from global memory (rows m = t*B + b) or from a CTA's shared-memory copy.
__device__ __forceinline__ void vtrace_trajectory(const VtraceCfg& cfg, const float* pol_base, int pol_stride,
                                                  const float* val_base, int val_stride, const Inputs& in,
                                                  const VtraceOut& out, float* __restrict__ dlogits,
                                                  float* __restrict__ dv, int b, int B, int T, int A, int lane,
                                                  float& l_pg, float& l_bl, float& l_en) {
  const int Tp = T - 2;
  const int t = lane;
  const bool live = t < T;
  const int m = live ? t * B + b : 0;       // time-major activation row
  const int src = live ? b * T + t : 0;     // batch-major input index
  const float* prow = pol_base + (size_t)(live ? t : 0) * pol_stride;
  float V = 0.f, rew = 0.f, gam = 0.f, rhob = 0.f, pi_a = 1.f;
  int act = 0;
  if (live) {
    V = val_base[(size_t)t * val_stride];
    act = in.action[src];
    rew = clip_reward(in.reward[src], cfg.reward_clipping);
    gam = in.done[src] ? 0.f : cfg.discount;                               // agent/impala.py:51
    const bool act_ok = act >= 0 && act < A;                                // tf.one_hot: an out-of-range index selects
    pi_a = act_ok ? prow[act] : 0.f;                                        // nothing (log(0), like the reference)
    const float mu_a = act_ok ? in.mu[(size_t)src * A + act] : 0.f;
    const float log_rho = logf(pi_a) - logf(mu_a);                         // optimizer/vtrace.py:46-51
    const float rho = expf(log_rho);                                       // :74
    rhob = fminf(1.0f, rho);                                               // :75-80 (clip_rho = cs = min(1, rho))
  }
  const float Vn = __shfl_down_sync(0xffffffffu, V, 1);
  const float delta = (t <= T - 2) ? rhob * (rew + gam * Vn - V) : 0.f;    // :84
  const float gc = gam * rhob;
  // window 1: steps 1..T-2 (bootstrap V_{T-1}); window 0: steps 0..T-3 (bootstrap V_{T-2})
  float a1 = (t <= T - 2) ? gc : 0.f, b1 = (t <= T - 2) ? delta : 0.f;
  float a0 = (t <= T - 3) ? gc : 0.f, b0 = (t <= T - 3) ? delta : 0.f;
  warp_affine_suffix_scan(a1, b1, lane);
  warp_affine_suffix_scan(a0, b0, lane);
  const float vs = V + b0;                                                 // :101
  const float vs1 = V + b1;
  const float vs1n = __shfl_down_sync(0xffffffffu, vs1, 1);               // vs_plus_1 at this step
  if (t < Tp) {
    const float adv = rhob * (rew + gam * vs1n - V);                       // agent/impala.py:78-80
    const size_t o = (size_t)b * Tp + t;
    out.vs[o] = vs;
    out.clipped_rho[o] = rhob;
    out.vs_plus_1[o] = vs1n;
    out.pg_adv[o] = adv;
    // losses (optimizer/vtrace.py:105-126)
    l_pg = -logf(pi_a + 1e-8f) * adv;
    const float err = vs - V;
    l_bl = 0.5f * err * err;
    // gradients wrt logits through softmax:  g_k = dL/dpi_k ; dlogit_k = pi_k (g_k - sum_j pi_j g_j)
    float s = 0.f, ent = 0.f;
    for (int k = 0; k < A; ++k) {
      const float p = prow[k];
      const float lp = logf(p);
      ent += p * lp;
      float g = cfg.entropy_coef * (lp + 1.0f);
      if (k == act) g -= adv / (p + 1e-8f);
      s += p * g;
    }
    l_en = ent;
    float* drow = dlogits + (size_t)m * 32;
    for (int k = 0; k < A; ++k) {
      const float p = prow[k];
      float g = cfg.entropy_coef * (logf(p) + 1.0f);
      if (k == act) g -= adv / (p + 1e-8f);
      drow[k] = p * (g - s);
    }
    dv[(size_t)m * 32] = -cfg.baseline_coef * err;
  }
}

__global__ void __launch_bounds__(128) vtrace_losses_kernel(
    VtraceCfg cfg, const float* __restrict__ policy, const float* __restrict__ value, Inputs in, VtraceOut out,
    float* __restrict__ dlogits, float* __restrict__ dv, int B, int T, int A) {
  kernel_prologue();
  __shared__ float red[4][3];
  __shared__ bool is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * 4 + warp;
  float l_pg = 0.f, l_bl = 0.f, l_en = 0.f;
  if (b < B)
    vtrace_trajectory(cfg, policy + (size_t)b * A, B * A, value + b, B, in, out, dlogits, dv, b, B, T, A, lane, l_pg,
                      l_bl, l_en);
  // ---- deterministic loss reduction: warp -> block -> last block sums the block partials -----
  l_pg = warp_sum(l_pg); l_bl = warp_sum(l_bl); l_en = warp_sum(l_en);
  if (lane == 0) { red[warp][0] = l_pg; red[warp][1] = l_bl; red[warp][2] = l_en; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float* p = out.loss_partials + (size_t)blockIdx.x * 3;
    for (int j = 0; j < 3; ++j) p[j] = (red[0][j] + red[1][j]) + (red[2][j] + red[3][j]);
    __threadfence();
    const unsigned int tk = atomicAdd(out.ticket, 1u);
    is_last = (tk == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && threadIdx.x < 3) {
    __threadfence();
    float acc = 0.f;
    for (unsigned int i = 0; i < gridDim.x; ++i) acc += out.loss_partials[(size_t)i * 3 + threadIdx.x];
    out.loss_sums[threadIdx.x] = acc;
    if (threadIdx.x == 0) *out.ticket = 0u;
  }
}

int vtrace_losses(cudaStream_t s, const VtraceCfg& cfg, const float* policy, const float* value, const Inputs& in,
                  const VtraceOut& out, float* dlogits, float* dv, int B, int T, int A) {
  if (T < 3 || T > 32) { set_error("trajectory %d outside [3,32]", T); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK((launch_k(vtrace_losses_kernel, cdiv(B, 4), 128, 0, s, cfg, policy, value, in, out, dlogits, dv, B, T, A)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// from_importance_weights (optimizer/vtrace.py:71-103), time-major [T,B]: one thread per b
// (consecutive lanes = consecutive b => every load/store is fully coalesced), the reverse scan
// runs in registers.  clip < 0 means clip_rho_threshold=None.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vtrace_fiw_kernel(const float* __restrict__ log_rhos,
                                                          const float* __restrict__ discounts,
                                                          const float* __restrict__ rewards,
                                                          const float* __restrict__ values,
                                                          const float* __restrict__ bootstrap, int T, int B,
                                                          float clip, float* __restrict__ vs,
                                                          float* __restrict__ clipped) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f;
  float vnext = bootstrap[b];
  constexpr int U = 4;
  int t = T - 1;
  for (; t - (U - 1) >= 0; t -= U) {   // issue U independent loads per array before the dependent chain
    float lr[U], g[U], r[U], v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const size_t o = (size_t)(t - u) * B + b;
      lr[u] = __ldg(log_rhos + o); g[u] = __ldg(discounts + o); r[u] = __ldg(rewards + o); v[u] = __ldg(values + o);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float rho = expf(lr[u]);
      const float rb = (clip >= 0.f) ? fminf(clip, rho) : rho;
      const float c = fminf(1.0f, rho);
      const float delta = rb * (r[u] + g[u] * vnext - v[u]);
      acc = delta + g[u] * c * acc;
      const size_t o = (size_t)(t - u) * B + b;
      vs[o] = acc + v[u];
      clipped[o] = rb;
      vnext = v[u];
    }
  }
  for (; t >= 0; --t) {
    const size_t o = (size_t)t * B + b;
    const float v = __ldg(values + o), g = __ldg(discounts + o);
    const float rho = expf(__ldg(log_rhos + o));
    const float rb = (clip >= 0.f) ? fminf(clip, rho) : rho;
    const float c = fminf(1.0f, rho);
    const float delta = rb * (__ldg(rewards + o) + g * vnext - v);
    acc = delta + g * c * acc;
    vs[o] = acc + v;
    clipped[o] = rb;
    vnext = v;
  }
}

// ------------------------------------------------------------------------------------------
// from_softmax (optimizer/vtrace.py:29-69), batch-major: one warp per trajectory.  The [T,A]
// behaviour/target softmax blocks of a trajectory are contiguous and are streamed with coalesced
// (float4 when aligned) loads into shared memory; lane = time step within a 32-step chunk, chunks
// are processed from the end of the trajectory with the scan carry passed between them.
// ------------------------------------------------------------------------------------------
constexpr int kFsWarps = 4;

__global__ void __launch_bounds__(kFsWarps * 32) vtrace_from_softmax_kernel(
    const float* __restrict__ mu, const float* __restrict__ pi, const int32_t* __restrict__ actions,
    const float* __restrict__ discounts, const float* __restrict__ rewards, const float* __restrict__ values,
    const float* __restrict__ next_values, int B, int T, int A, float clip, float* __restrict__ vs,
    float* __restrict__ clipped) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kFsWarps + warp;
  if (b >= B) return;
  const int chunkA = 32 * A;                    // floats per 32-step chunk
  float* s_pi = sm + (size_t)warp * 2 * chunkA;
  float* s_mu = s_pi + chunkA;
  const size_t base = (size_t)b * T;
  const float boot = next_values[base + T - 1];                               // optimizer/vtrace.py:62
  float carry = 0.f;
  for (int t0 = ((T - 1) / 32) * 32; t0 >= 0; t0 -= 32) {
    const int nt = min(32, T - t0);
    const int nel = nt * A;
    const float* gpi = pi + (base + t0) * A;
    const float* gmu = mu + (base + t0) * A;
    if ((((size_t)gpi | (size_t)gmu) & 15) == 0 && (nel & 3) == 0) {
      for (int i = lane; i < nel / 4; i += 32) {
        reinterpret_cast<float4*>(s_pi)[i] = __ldg(reinterpret_cast<const float4*>(gpi) + i);
        reinterpret_cast<float4*>(s_mu)[i] = __ldg(reinterpret_cast<const float4*>(gmu) + i);
      }
    } else {
      for (int i = lane; i < nel; i += 32) { s_pi[i] = __ldg(gpi + i); s_mu[i] = __ldg(gmu + i); }
    }
    __syncwarp();
    const int t = t0 + lane;
    float a = 1.f, d = 0.f, v = 0.f, rb = 0.f;   // dead lanes carry the identity map
    if (lane < nt) {
      const int act = actions[base + t];
      float pa = 0.f, ma = 0.f;
      if (act >= 0 && act < A) { pa = s_pi[lane * A + act]; ma = s_mu[lane * A + act]; }   // tf.one_hot semantics
      const float rho = expf(logf(pa) - logf(ma));
      rb = (clip >= 0.f) ? fminf(clip, rho) : rho;
      const float c = fminf(1.0f, rho);
      v = values[base + t];
      const float vn = (t + 1 < T) ? values[base + t + 1] : boot;
      const float g = discounts[base + t];
      d = rb * (rewards[base + t] + g * vn - v);
      a = g * c;
    }
    warp_affine_suffix_scan(a, d, lane);
    const float acc = fmaf(a, carry, d);
    if (lane < nt) {
      vs[base + t] = acc + v;
      clipped[base + t] = rb;
    }
    carry = __shfl_sync(0xffffffffu, acc, 0);
    __syncwarp();
  }
}

// Fast path of from_softmax for the learner's shape class (T <= 32, 16-byte aligned [T,A] blocks): persistent
// warps, each looping over trajectories with a 2-stage cp.async pipeline -- the 16-byte global->shared copies of
// trajectory b+stride are in flight (no registers, L1 bypass) while trajectory b is scanned, and the five
// per-step scalars of the next trajectory are prefetched into registers.
__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)),
               "l"(gmem_src)
               : "memory");
}
__global__ void __launch_bounds__(kFsWarps * 32) vtrace_from_softmax_pipe_kernel(
    const float* __restrict__ mu, const float* __restrict__ pi, const int32_t* __restrict__ actions,
    const float* __restrict__ discounts, const float* __restrict__ rewards, const float* __restrict__ values,
    const float* __restrict__ next_values, int B, int T, int A, float clip, float* __restrict__ vs,
    float* __restrict__ clipped) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int TA = T * A;                               // multiple of 4 (checked by the launcher)
  float* wbase = sm + (size_t)warp * 4 * TA;          // [stage][pi|mu][TA]
  const int nwarps = gridDim.x * kFsWarps;
  int b = blockIdx.x * kFsWarps + warp;
  if (b >= B) return;

  auto issue = [&](int bb, int stage) {
    float* s_pi = wbase + stage * 2 * TA;
    float* s_mu = s_pi + TA;
    const float* gpi = pi + (size_t)bb * TA;
    const float* gmu = mu + (size_t)bb * TA;
    for (int i = lane; i < TA / 4; i += 32) {
      cp_async16(s_pi + 4 * i, gpi + 4 * i);
      cp_async16(s_mu + 4 * i, gmu + 4 * i);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  struct Scal { int act; float g, r, v, vn; };
  auto scalars = [&](int bb) {
    Scal s{0, 0.f, 0.f, 0.f, 0.f};
    if (lane < T) {
      const size_t o = (size_t)bb * T + lane;
      s.act = __ldg(actions + o);
      s.g = __ldg(discounts + o);
      s.r = __ldg(rewards + o);
      s.v = __ldg(values + o);
      s.vn = (lane + 1 < T) ? __ldg(values + o + 1) : __ldg(next_values + (size_t)bb * T + T - 1);
    }
    return s;
  };

  issue(b, 0);
  Scal cur = scalars(b);
  int stage = 0;
  for (; b < B; b += nwarps) {
    const int nb = b + nwarps;
    Scal nxt{0, 0.f, 0.f, 0.f, 0.f};
    if (nb < B) {
      issue(nb, stage ^ 1);
      nxt = scalars(nb);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncwarp();
    const float* s_pi = wbase + stage * 2 * TA;
    const float* s_mu = s_pi + TA;
    float a = 1.f, d = 0.f, rb = 0.f;
    if (lane < T) {
      float pa = 0.f, ma = 0.f;
      if (cur.act >= 0 && cur.act < A) { pa = s_pi[lane * A + cur.act]; ma = s_mu[lane * A + cur.act]; }
      const float rho = expf(logf(pa) - logf(ma));
      rb = (clip >= 0.f) ? fminf(clip, rho) : rho;
      const float c = fminf(1.0f, rho);
      d = rb * (cur.r + cur.g * cur.vn - cur.v);
      a = cur.g * c;
    }
    warp_affine_suffix_scan(a, d, lane);
    if (lane < T) {
      const size_t o = (size_t)b * T + lane;
      vs[o] = d + cur.v;
      clipped[o] = rb;
    }
    cur = nxt;
    stage ^= 1;
    __syncwarp();      // everyone is done reading this stage before the next issue() overwrites it
  }
}

static int launch_fiw(cudaStream_t s, const float* lr, const float* g, const float* r, const float* v,
                      const float* boot, int T, int B, float clip, float* vs, float* cl) {
  if (T < 1 || B < 1) { set_error("vtrace: T and B must be positive"); return DRL_ERR_INVALID; }
  vtrace_fiw_kernel<<<cdiv(B, 256), 256, 0, s>>>(lr, g, r, v, boot, T, B, clip, vs, cl);
  DRL_CHECK_LAUNCH();
  return DRL_OK;
}

static int launch_fs(cudaStream_t s, const float* mu, const float* pi, const int32_t* a, const float* g,
                     const float* r, const float* v, const float* nv, int B, int T, int A, float clip, float* vs,
                     float* cl) {
  if (T < 1 || B < 1 || A < 1) { set_error("vtrace: B, T, A must be positive"); return DRL_ERR_INVALID; }
  // learner-shaped fast path: persistent warps with a cp.async pipeline
  const size_t smem_pipe = (size_t)kFsWarps * 4 * T * A * sizeof(float);
  if (T <= 32 && ((T * A) & 3) == 0 && ((((size_t)mu | (size_t)pi)) & 15) == 0 && smem_pipe <= 48 * 1024) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(12, (200 * 1024) / std::max<size_t>(smem_pipe, 1)));
    const int grid = std::min(cdiv(B, kFsWarps), sms * per_sm);
    vtrace_from_softmax_pipe_kernel<<<grid, kFsWarps * 32, smem_pipe, s>>>(mu, pi, a, g, r, v, nv, B, T, A, clip, vs, cl);
    DRL_CHECK_LAUNCH();
    return DRL_OK;
  }
  const size_t smem = (size_t)kFsWarps * 2 * 32 * A * sizeof(float);
  if (smem > 200 * 1024) { set_error("vtrace: action_size %d too large", A); return DRL_ERR_INVALID; }
  static size_t smem_set = 0;
  if (smem > 48 * 1024 && smem > smem_set) {
    DRL_CUDA_CHECK(cudaFuncSetAttribute(vtrace_from_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
    smem_set = smem;
  }
  vtrace_from_softmax_kernel<<<cdiv(B, kFsWarps), kFsWarps * 32, smem, s>>>(mu, pi, a, g, r, v, nv, B, T, A, clip, vs,
                                                                            cl);
  DRL_CHECK_LAUNCH();
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// Stand-alone loss sums (optimizer/vtrace.py:105-126) + log pi(a) (:16-27): one thread per (b,t),
// block partials written to `partials` [gridDim.x, 3] and summed on the host in block order.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vtrace_loss_sums_kernel(const float* __restrict__ sm,
                                                                const int32_t* __restrict__ actions,
                                                                const float* __restrict__ adv,
                                                                const float* __restrict__ vs,
                                                                const float* __restrict__ value, int n, int A,
                                                                float* __restrict__ partials,
                                                                float* __restrict__ log_probs) {
  __shared__ float red[8][3];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float pg = 0.f, bl = 0.f, en = 0.f;
  if (i < n) {
    const float* row = sm + (size_t)i * A;
    const int a = actions[i];
    float sel = 0.f;
    for (int k = 0; k < A; ++k) {
      const float p = row[k];
      en += p * logf(p);
      if (k == a) sel = p;
    }
    if (log_probs) log_probs[i] = logf(sel);
    pg = -logf(sel + 1e-8f) * adv[i];
    const float e = vs[i] - value[i];
    bl = 0.5f * e * e;
  }
  pg = warp_sum(pg); bl = warp_sum(bl); en = warp_sum(en);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[warp][0] = pg; red[warp][1] = bl; red[warp][2] = en; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    partials[(size_t)blockIdx.x * 3 + threadIdx.x] = s;
  }
}

// small RAII helper for the host-pointer convenience entry points
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t bytes) { DRL_CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 4)); return DRL_OK; }
  int upload(const void* h, size_t bytes) {
    DRL_TRY(alloc(bytes));
    DRL_CUDA_CHECK(cudaMemcpy(p, h, bytes, cudaMemcpyHostToDevice));
    return DRL_OK;
  }
  template <class T> T* as() { return static_cast<T*>(p); }
};

}  // namespace drl

using namespace drl;

extern "C" {

int drl_vtrace_from_importance_weights_dev(const float* log_rhos, const float* discounts, const float* rewards,
                                           const float* values, const float* bootstrap_value, int32_t T, int32_t B,
                                           float clip_rho_threshold, float* vs, float* clipped_rhos, void* stream) {
  return launch_fiw(static_cast<cudaStream_t>(stream), log_rhos, discounts, rewards, values, bootstrap_value, T, B,
                    clip_rho_threshold, vs, clipped_rhos);
}

int drl_vtrace_from_importance_weights(const float* log_rhos, const float* discounts, const float* rewards,
                                       const float* values, const float* bootstrap_value, int32_t T, int32_t B,
                                       float clip_rho_threshold, float* vs, float* clipped_rhos) {
  if (!log_rhos || !discounts || !rewards || !values || !bootstrap_value || !vs || !clipped_rhos) {
    set_error("vtrace: null pointer");
    return DRL_ERR_INVALID;
  }
  if (T < 1 || B < 1) { set_error("vtrace: T and B must be positive"); return DRL_ERR_INVALID; }
  const size_t n = (size_t)T * B * sizeof(float);
  DevBuf a, b, c, d, e, o1, o2;
  DRL_TRY(a.upload(log_rhos, n)); DRL_TRY(b.upload(discounts, n)); DRL_TRY(c.upload(rewards, n));
  DRL_TRY(d.upload(values, n)); DRL_TRY(e.upload(bootstrap_value, (size_t)B * sizeof(float)));
  DRL_TRY(o1.alloc(n)); DRL_TRY(o2.alloc(n));
  DRL_TRY(launch_fiw(0, a.as<float>(), b.as<float>(), c.as<float>(), d.as<float>(), e.as<float>(), T, B,
                     clip_rho_threshold, o1.as<float>(), o2.as<float>()));
  DRL_CUDA_CHECK(cudaMemcpy(vs, o1.p, n, cudaMemcpyDeviceToHost));
  DRL_CUDA_CHECK(cudaMemcpy(clipped_rhos, o2.p, n, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_vtrace_from_softmax_dev(const float* mu, const float* pi, const int32_t* actions, const float* discounts,
                                const float* rewards, const float* values, const float* next_values, int32_t B,
                                int32_t T, int32_t A, float clip_rho_threshold, float* vs, float* clipped_rho,
                                void* stream) {
  return launch_fs(static_cast<cudaStream_t>(stream), mu, pi, actions, discounts, rewards, values, next_values, B, T,
                   A, clip_rho_threshold, vs, clipped_rho);
}

int drl_vtrace_from_softmax(const float* mu, const float* pi, const int32_t* actions, const float* discounts,
                            const float* rewards, const float* values, const float* next_values, int32_t B, int32_t T,
                            int32_t A, float clip_rho_threshold, float* vs, float* clipped_rho) {
  if (!mu || !pi || !actions || !discounts || !rewards || !values || !next_values || !vs || !clipped_rho) {
    set_error("vtrace: null pointer");
    return DRL_ERR_INVALID;
  }
  if (T < 1 || B < 1 || A < 1) { set_error("vtrace: B, T, A must be positive"); return DRL_ERR_INVALID; }
  const size_t n = (size_t)B * T * sizeof(float);
  DevBuf dmu, dpi, da, dg, dr, dv, dnv, o1, o2;
  DRL_TRY(dmu.upload(mu, n * A)); DRL_TRY(dpi.upload(pi, n * A)); DRL_TRY(da.upload(actions, n));
  DRL_TRY(dg.upload(discounts, n)); DRL_TRY(dr.upload(rewards, n)); DRL_TRY(dv.upload(values, n));
  DRL_TRY(dnv.upload(next_values, n));
  DRL_TRY(o1.alloc(n)); DRL_TRY(o2.alloc(n));
  DRL_TRY(launch_fs(0, dmu.as<float>(), dpi.as<float>(), da.as<int32_t>(), dg.as<float>(), dr.as<float>(),
                    dv.as<float>(), dnv.as<float>(), B, T, A, clip_rho_threshold, o1.as<float>(), o2.as<float>()));
  DRL_CUDA_CHECK(cudaMemcpy(vs, o1.p, n, cudaMemcpyDeviceToHost));
  DRL_CUDA_CHECK(cudaMemcpy(clipped_rho, o2.p, n, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_vtrace_loss_sums(const float* softmax, const int32_t* actions, const float* advantages, const float* vs,
                         const float* value, int32_t B, int32_t T, int32_t A, float* sums, float* log_probs) {
  if (!softmax || !actions || !advantages || !vs || !value || !sums) { set_error("loss_sums: null pointer"); return DRL_ERR_INVALID; }
  if (T < 1 || B < 1 || A < 1) { set_error("loss_sums: B, T, A must be positive"); return DRL_ERR_INVALID; }
  const int n = B * T;
  const size_t nb = (size_t)n * sizeof(float);
  const int nblk = cdiv(n, 256);
  DevBuf dsm, da, dadv, dvs, dval, dpart, dlp;
  DRL_TRY(dsm.upload(softmax, nb * A)); DRL_TRY(da.upload(actions, nb)); DRL_TRY(dadv.upload(advantages, nb));
  DRL_TRY(dvs.upload(vs, nb)); DRL_TRY(dval.upload(value, nb));
  DRL_TRY(dpart.alloc((size_t)nblk * 3 * sizeof(float))); DRL_TRY(dlp.alloc(nb));
  vtrace_loss_sums_kernel<<<nblk, 256>>>(dsm.as<float>(), da.as<int32_t>(), dadv.as<float>(), dvs.as<float>(),
                                         dval.as<float>(), n, A, dpart.as<float>(), dlp.as<float>());
  DRL_CHECK_LAUNCH();
  std::vector<float> part((size_t)nblk * 3);
  DRL_CUDA_CHECK(cudaMemcpy(part.data(), dpart.p, part.size() * sizeof(float), cudaMemcpyDeviceToHost));
  if (log_probs) DRL_CUDA_CHECK(cudaMemcpy(log_probs, dlp.p, nb, cudaMemcpyDeviceToHost));
  for (int j = 0; j < 3; ++j) {
    float s = 0.f;
    for (int b = 0; b < nblk; ++b) s += part[(size_t)b * 3 + j];
    sums[j] = s;
  }
  return DRL_OK;
}

}  // extern "C"
