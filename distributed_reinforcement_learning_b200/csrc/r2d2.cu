// r2d2.cu -- the R2D2 learner behind drl_r2d2_* (include/drl_b200.h): replaces r2d2.Agent's learner graph
// (agent/r2d2.py:13-95) over model/r2d2_lstm.py:28-116 (stored-state LSTM unroll, main and target scope),
// optimizer/burn_in.py:23-32 (value-function rescaling) and TF1 Adam.
//
// The reference unrolls `network` seq_len times per scope with the carried (h, c) multiplied by (1 - done_i) after
// step i (model/r2d2_lstm.py:67-84).  Only the LSTM cell is sequential: the convolutions, the action embedding and
// the input half of the LSTM contraction ([a3 | emb] W_x, 3392 of the 3456 kernel rows) do not depend on the carried
// state, so they run over all M = B*S rows at once through the same gather-GEMM kernels as the IMPALA learner
// (time-major rows m = t*B + b).  What remains per step is h_{t-1} W_h (64 x 256) + the gate nonlinearity: one
// persistent CTA per sequence keeps W_h in shared memory and walks the S steps (r2d2_lstm_fwd_kernel); BPTT is the
// mirror image (r2d2_lstm_bwd_kernel, W_h^T in shared memory), after which every weight / data gradient is again one
// batched GEMM over all M rows (all rows receive gradient: burn-in only slices the loss, agent/r2d2.py:64-68).
// That holds at lstm_size 64; at 256 and 512, W_h (1 MB / 4 MB) is spread over a thread-block cluster instead
// (r2d2_cluster.cuh), and the GEMMs take the width at run time.
#include <string.h>

#include <algorithm>

#include <string>
#include <vector>

#include "adam_learner.cuh"
#include "layer_defs.cuh"
#include "r2d2_cluster.cuh"
#include "r2d2_defs.cuh"

namespace drl {

// step input [a3 | emb[prev_action]] with the (t,b) -> (b,t) remap of prev_action (K = 3392)
struct R2XA {
  static constexpr bool kContigK = true;
  const float* e; const float* table; const int* pa; RowMap map;
  struct Row { const float *pe, *pu; };
  __device__ __forceinline__ Row row(int, int m) const {
    Row r;
    if (m < 0) { r.pe = nullptr; r.pu = nullptr; return r; }
    r.pe = e + (size_t)m * Geo::FLAT;
    r.pu = table + (size_t)__ldg(pa + map.src(m)) * Geo::EMB;
    return r;
  }
  __device__ __forceinline__ float4 load(const Row& r, int k) const {
    if (r.pe == nullptr) return zero4();
    return __ldg(reinterpret_cast<const float4*>((k < Geo::FLAT) ? r.pe + k : r.pu + (k - Geo::FLAT)));
  }
};

// split-K plan of lstm_x_fwd ([M, 3392] x [3392, G = 4L]): about one wave over the M x N tiles (N: one 256-wide tensor-core
// tile at L = 64, 4 or 8 at 256 / 512)
static SplitPlan plan_r2_x(int M, int mode, int G) {
  return mode >= 2 ? plan_split(kR2Cat, cdiv(M, 128) * cdiv(G, 256), 32, 1)
                   : plan_split(kR2Cat, cdiv(M, CfgMid::BM) * (G / CfgMid::BN), 16, 1);
}

// ------------------------------------------------------------------------------------------
// LSTM recurrence, forward (model/r2d2_lstm.py:12-21 inside the unroll :67-84; TF 1.14 LSTMCell):
//   z_t = sum_s zpart[s][m] + b + h_in W_h ; i,j,f,o = split(z_t)
//   c_t = sigmoid(f + 1) c_in + sigmoid(i) tanh(j) ; h_t = sigmoid(o) tanh(c_t)         (h_t feeds the q head)
//   (h_in, c_in) of step t+1 = (h_t, c_t) * (1 - done_t)
// One CTA per sequence, 4L = 256 threads; thread j owns gate column j and keeps W_h[:, j] (L = 64 floats) in REGISTERS for
// all S steps: with W_h in shared memory every step re-read its 64 KB (512 clk of LDS bandwidth per SM, measured
// 1.36 us per step); from registers a step costs 16 broadcast LDS.128 of h plus 64 FMAs per thread.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kR2G) r2d2_lstm_fwd_kernel(
    const float* __restrict__ zpart, int nsplit, size_t slab, const float* __restrict__ bias,
    const float* __restrict__ Wh, const float* __restrict__ h0, const float* __restrict__ c0,
    const uint8_t* __restrict__ done, float* __restrict__ gates, float* __restrict__ tc, float* __restrict__ hout,
    float* __restrict__ hin, float* __restrict__ cin, float* __restrict__ c_last, int B, int S) {
  kernel_prologue();
  __shared__ __align__(16) float sh[kR2L];
  __shared__ float sz[kR2G];
  const int b = blockIdx.x, j = threadIdx.x;
  float w[kR2L];
#pragma unroll
  for (int k = 0; k < kR2L; ++k) w[k] = Wh[k * kR2G + j];      // coalesced across the CTA, once
  float c_reg = 0.f;
  if (j < kR2L) { sh[j] = h0[(size_t)b * kR2L + j]; c_reg = c0[(size_t)b * kR2L + j]; }
  const float bj = bias[j];
  // the step input z_x[t] and done[t] do not depend on the recurrence: the loads of step t+1 are issued at the top of
  // step t so that their latency (L2 / HBM) is off the serial chain
  auto load_z = [&](int t) {
    const size_t m = (size_t)t * B + b;
    float z = 0.f;
    for (int s = 0; s < nsplit; ++s) z += zpart[(size_t)s * slab + m * kR2G + j];
    return z;
  };
  float z_next = load_z(0);
  float keep_next = (done && done[(size_t)b * S]) ? 0.f : 1.f;
  __syncthreads();
  for (int t = 0; t < S; ++t) {
    const size_t m = (size_t)t * B + b;
    const float z = bj + z_next;
    const float keep = keep_next;
    if (t + 1 < S) {
      z_next = load_z(t + 1);
      keep_next = (done && done[(size_t)b * S + t + 1]) ? 0.f : 1.f;
    }
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;      // four independent chains: 16 dependent FMAs each
#pragma unroll
    for (int k = 0; k < kR2L; k += 4) {
      const float4 h4 = *reinterpret_cast<const float4*>(sh + k);     // broadcast
      acc0 = fmaf(h4.x, w[k], acc0);
      acc1 = fmaf(h4.y, w[k + 1], acc1);
      acc2 = fmaf(h4.z, w[k + 2], acc2);
      acc3 = fmaf(h4.w, w[k + 3], acc3);
    }
    // every thread applies the nonlinearity of its own gate column (warp-uniform branch: L = 2 warps per gate), so
    // the serial tail below is left with one tanh instead of five transcendentals
    const float pre = z + ((acc0 + acc1) + (acc2 + acc3));
    const int gate = j / kR2L;
    const float actv = (gate == 1) ? tanhf(pre) : sigmoidf_acc(gate == 2 ? pre + 1.0f : pre);
    sz[j] = actv;
    gates[m * kR2G + j] = actv;
    if (j < kR2L) { hin[m * kR2L + j] = sh[j]; cin[m * kR2L + j] = c_reg; }
    __syncthreads();
    if (j < kR2L) {
      const float si = sz[j], tj = sz[kR2L + j], sf = sz[2 * kR2L + j], so = sz[3 * kR2L + j];
      const float c = sf * c_reg + si * tj;
      const float tcv = tanhf(c);
      const float h = so * tcv;
      tc[m * kR2L + j] = tcv;
      hout[m * kR2L + j] = h;
      if (c_last) c_last[m * kR2L + j] = c;
      c_reg = c * keep;
      sh[j] = h * keep;
    }
    __syncthreads();
  }
}

// BPTT through the same recurrence (rows of all S steps receive gradient):
//   dh_t = dhout[m] + (1 - done_t) dh_in[t+1] ; dc_t = (1 - done_t) dc_in[t+1] + dh_t so (1 - tc^2)
//   do = dh_t tc so(1-so) ; di = dc_t tj si(1-si) ; dj = dc_t si (1 - tj^2) ; df = dc_t c_in sf(1-sf)
//   dc_in[t] = dc_t sf ; dh_in[t] = dz_t W_h^T        (the weights again live in registers, 64 per thread)
__global__ void __launch_bounds__(kR2G) r2d2_lstm_bwd_kernel(
    const float* __restrict__ dhout, const float* __restrict__ gates, const float* __restrict__ tc,
    const float* __restrict__ cin, const float* __restrict__ Wh, const uint8_t* __restrict__ done,
    float* __restrict__ dz, int B, int S) {
  kernel_prologue();
  __shared__ __align__(16) float sdz[kR2G];
  __shared__ float sdh[kR2L];
  __shared__ float spart[4 * kR2L];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int kk = tid & (kR2L - 1), q = tid / kR2L;
  // thread (kk, q) accumulates dh_in[kk] over gate columns [q L, (q+1) L): its 64 weights W_h[kk][q L + i] stay in registers
  float w[kR2L];
#pragma unroll
  for (int i = 0; i < kR2L; ++i) w[i] = Wh[(size_t)kk * kR2G + q * kR2L + i];
  float dc_carry = 0.f;
  if (tid < kR2L) sdh[tid] = 0.f;
  __syncthreads();
  // operands of step t-1 are fetched while step t computes (they do not depend on the recurrence)
  struct Ops { float dho, si, tj, sf, so, tcv, cprev, keep; };
  auto fetch = [&](int t) {
    Ops o{};
    if (tid < kR2L) {
      const size_t m = (size_t)t * B + b;
      const float* g = gates + m * kR2G;
      o.dho = dhout[m * kR2L + tid];
      o.si = g[tid]; o.tj = g[kR2L + tid]; o.sf = g[2 * kR2L + tid]; o.so = g[3 * kR2L + tid];
      o.tcv = tc[m * kR2L + tid];
      o.cprev = cin[m * kR2L + tid];
      o.keep = done[(size_t)b * S + t] ? 0.f : 1.f;
    }
    return o;
  };
  Ops nxt = fetch(S - 1);
  for (int t = S - 1; t >= 0; --t) {
    const size_t m = (size_t)t * B + b;
    const Ops cur = nxt;
    if (t > 0) nxt = fetch(t - 1);
    if (tid < kR2L) {
      const float keep = cur.keep;
      const float dh = cur.dho + keep * sdh[tid];
      const float si = cur.si, tj = cur.tj, sf = cur.sf, so = cur.so;
      const float tcv = cur.tcv;
      const float cprev = cur.cprev;
      const float d_o = dh * tcv * so * (1.f - so);
      const float dc = keep * dc_carry + dh * so * (1.f - tcv * tcv);
      const float di = dc * tj * si * (1.f - si);
      const float dj = dc * si * (1.f - tj * tj);
      const float df = dc * cprev * sf * (1.f - sf);
      sdz[tid] = di; sdz[kR2L + tid] = dj; sdz[2 * kR2L + tid] = df; sdz[3 * kR2L + tid] = d_o;
      dc_carry = dc * sf;
    }
    __syncthreads();
    dz[m * kR2G + tid] = sdz[tid];                    // coalesced store of the step's 4L gate gradients
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
#pragma unroll
    for (int i = 0; i < kR2L; i += 4) {
      const float4 d4 = *reinterpret_cast<const float4*>(sdz + q * kR2L + i);   // broadcast within the warp
      acc0 = fmaf(d4.x, w[i], acc0);
      acc1 = fmaf(d4.y, w[i + 1], acc1);
      acc2 = fmaf(d4.z, w[i + 2], acc2);
      acc3 = fmaf(d4.w, w[i + 3], acc3);
    }
    spart[q * kR2L + kk] = (acc0 + acc1) + (acc2 + acc3);
    __syncthreads();
    // sdh[tid] is only read by the thread that writes it; spart / sdz are protected by the two barriers above
    if (tid < kR2L) sdh[tid] = (spart[tid] + spart[kR2L + tid]) + (spart[2 * kR2L + tid] + spart[3 * kR2L + tid]);
  }
}

// q[m][a] = (q1[m] Wv[:, a] + bv[a]) - (q1[m] wm + bm)      (model/r2d2_lstm.py:51-53); one warp per row
__global__ void __launch_bounds__(128) r2d2_out_kernel(const float* __restrict__ q1, const float* __restrict__ wv,
                                                        const float* __restrict__ bv, const float* __restrict__ wm,
                                                        const float* __restrict__ bm, float* __restrict__ q, int M, int A) {
  kernel_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  if (m >= M) return;
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = q1[(size_t)m * kR2H + lane + 32 * i];
  float mean = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) mean = fmaf(x[i], __ldg(wm + lane + 32 * i), mean);
  mean = warp_sum(mean) + bm[0];
  for (int a = 0; a < A; ++a) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) v = fmaf(x[i], __ldg(wv + (size_t)(lane + 32 * i) * A + a), v);
    v = warp_sum(v);
    if (lane == 0) q[(size_t)m * A + a] = (v + bv[a]) - mean;
  }
}

// dq1[m][k] = relu'(q1) (sum_a dq[m][a] Wv[k][a] + dmean[m] wm[k]);  grid = rows, 128 threads
__global__ void __launch_bounds__(kR2H) r2d2_out_bwd_kernel(const float* __restrict__ dq, const float* __restrict__ dmean,
                                                             const float* __restrict__ wv, const float* __restrict__ wm,
                                                             const float* __restrict__ q1, float* __restrict__ dq1, int A) {
  kernel_prologue();
  __shared__ float sd[32];
  __shared__ float sdm;
  const int m = blockIdx.x, k = threadIdx.x;
  if (k < A) sd[k] = dq[(size_t)m * 32 + k];
  if (k == 0) sdm = dmean[(size_t)m * 32];
  __syncthreads();
  float acc = sdm * __ldg(wm + k);
  for (int a = 0; a < A; ++a) acc = fmaf(sd[a], __ldg(wv + (size_t)k * A + a), acc);
  const size_t o = (size_t)m * kR2H + k;
  dq1[o] = (q1[o] > 0.f) ? acc : 0.f;
}

// ------------------------------------------------------------------------------------------
// TD targets, loss and head gradients (agent/r2d2.py:62-90), window i in [0, Nt), t = burn_in + i, Nt = S - burn_in - 1:
//   sav = main_q[b,t][action[b,t]] ; next_action = argmax main_q[b,t+1] (first maximum) ; nsav = target_q[b,t+1][next_action]
//   target = h(h^-1(nsav) * gamma (1 - done[b,t]) + reward[b,t])        (h = value_function_rescaling, eps 1e-3)
//   loss = mean_b w_b mean_i (target - sav)^2 ; td[b] = |mean_i (target - sav)|
// The two rescalings are evaluated in float64: h^-1 subtracts 1 from sqrt(1 + 4 eps (..)) ~ 1.002, which costs float32
// three digits.  One block; a warp owns sequences b = warp, warp + 8, ...; all reductions in a fixed order.
// NSTEP (r2d2_td_nstep_kernel, DESIGN.md section 22): the n-step double-Q target over k = min(n, S - 1 - t) steps,
//   G = sum_{j<k} (prod_{l<j} D_{t+l}) r[t+j] + (prod_{l<k} D_{t+l}) h^-1(target_q[t+k][argmax main_q[t+k]]),
//   D = gamma (1 - done), target = h(G), all in float64; and, when `mixed`, the priority
//   td[b] = eta max_i |diff| + (1 - eta) mean_i |diff| instead of |mean_i diff|.  At k = 1 the target expression is the
//   one-step one term for term (G = r exactly), so n = 1 reproduces its bits.
// ------------------------------------------------------------------------------------------
struct R2TdArgs {
  const float* mq; const float* tq;            // [M, A] time-major
  const int32_t* action; const float* reward; const uint8_t* done; const float* weight;   // batch-major; weight may be null
  float discount; int B, S, burn_in, A;
  float* sav; float* target_value;             // [B, Nt] taps
  float* td_dev; float* td_host;               // [B]
  float* dq; float* dmean;                     // [M, 32] or null
  float* loss;                                 // [1] or null
};
__device__ __forceinline__ double r2_h(double x) {
  const double s = (x > 0.0) - (x < 0.0);
  return s * (sqrt(fabs(x) + 1.0) - 1.0) + 1e-3 * x;
}
__device__ __forceinline__ double r2_hinv(double x) {
  const double s = (x > 0.0) - (x < 0.0);
  const double r = (sqrt(1.0 + 4.0 * 1e-3 * (fabs(x) + 1.0 + 1e-3)) - 1.0) / (2.0 * 1e-3);
  return s * (r * r - 1.0);
}
template <bool NSTEP>
__device__ __forceinline__ void r2d2_td_body(const R2TdArgs& a, int n, bool mixed, float eta) {
  kernel_prologue();
  __shared__ float red[8];
  const int Nt = a.S - a.burn_in - 1;
  const int M = a.B * a.S;
  if (a.dq) {      // rows outside the loss window carry no gradient; columns >= A / >= 1 are never written (stay zero)
    const int W = a.A + 1;
    for (int i = threadIdx.x; i < M * W; i += blockDim.x) {
      const int m = i / W, k = i - m * W;
      if (k < a.A) a.dq[(size_t)m * 32 + k] = 0.f;
      else a.dmean[(size_t)m * 32] = 0.f;
    }
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float wloss = 0.f;
  for (int b = warp; b < a.B; b += 8) {
    const float w = a.weight ? a.weight[b] : 1.0f;
    float sdiff = 0.f, ssq = 0.f, sabs = 0.f, mabs = 0.f;
    for (int i = lane; i < Nt; i += 32) {
      const int t = a.burn_in + i;
      const size_t m = (size_t)t * a.B + b, mn = (size_t)(t + 1) * a.B + b;
      // NSTEP: the bootstrap row is t + k, the horizon k = min(n, S - 1 - t) cut at the last step of the sequence
      const size_t mb = NSTEP ? (size_t)(t + min(n, a.S - 1 - t)) * a.B + b : mn;
      const int act = a.action[(size_t)b * a.S + t];
      float best = -INFINITY;
      int arg = 0;
      for (int k = 0; k < a.A; ++k) {
        const float v = a.mq[mb * a.A + k];
        if (v > best) { best = v; arg = k; }
      }
      const bool act_ok = act >= 0 && act < a.A;            // tf.one_hot: an out-of-range action selects nothing
      const float sav = act_ok ? a.mq[m * a.A + act] : 0.f;
      const float nsav = a.tq[mb * a.A + arg];
      float target;
      if constexpr (NSTEP) {
        const size_t r0 = (size_t)b * a.S + t;
        const int hz = min(n, a.S - 1 - t);
        double ret = 0.0, disc = 1.0;        // sum_{j<k} (prod_{l<j} D) r[t+j], then prod_{l<k} D
        for (int j = 0; j < hz; ++j) {
          ret += disc * (double)a.reward[r0 + j];
          disc *= a.done[r0 + j] ? 0.0 : (double)a.discount;
        }
        target = (float)r2_h(r2_hinv((double)nsav) * disc + ret);
      } else {
        const double disc = a.done[(size_t)b * a.S + t] ? 0.0 : (double)a.discount;
        target = (float)r2_h(r2_hinv((double)nsav) * disc + (double)a.reward[(size_t)b * a.S + t]);
      }
      const float diff = target - sav;
      a.sav[(size_t)b * Nt + i] = sav;
      a.target_value[(size_t)b * Nt + i] = target;
      sdiff += diff;
      ssq += diff * diff;
      if (NSTEP && mixed) {
        sabs += fabsf(diff);
        mabs = fmaxf(mabs, fabsf(diff));
      }
      if (a.dq) {
        const float g = -2.0f * w * diff / ((float)Nt * (float)a.B);
        if (act_ok) {
          a.dq[m * 32 + act] = g;
          a.dmean[m * 32] = -g;
        }
      }
    }
    sdiff = warp_sum(sdiff);
    ssq = warp_sum(ssq);
    if (NSTEP && mixed) {
      sabs = warp_sum(sabs);
      mabs = warp_max(mabs);
    }
    if (lane == 0) {
      const float td = (NSTEP && mixed) ? eta * mabs + (1.0f - eta) * (sabs / (float)Nt) : fabsf(sdiff / (float)Nt);
      a.td_dev[b] = td;
      if (a.td_host) a.td_host[b] = td;
      wloss += w * (ssq / (float)Nt);
    }
  }
  if (a.loss) {
    if (lane == 0) red[warp] = wloss;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += red[i];
      *a.loss = s / (float)a.B;
    }
  }
}
__global__ void __launch_bounds__(256) r2d2_td_kernel(R2TdArgs a) {
  r2d2_td_body<false>(a, 1, false, 0.f);
}
// n >= 1; mixed: the priority rule eta max |diff| + (1 - eta) mean |diff| (eta in [0, 1]), otherwise |mean diff|
__global__ void __launch_bounds__(256) r2d2_td_nstep_kernel(R2TdArgs a, int n, int mixed, float eta) {
  r2d2_td_body<true>(a, n, mixed != 0, eta);
}


constexpr size_t kR2FwdSmem = 0, kR2BwdSmem = 0;     // the recurrence kernels only use small static shared arrays

int policy_conv_forward_tf32(cudaStream_t s, const TrunkLayout& pl, const float* P, const uint8_t* img_conv2,
                             const uint8_t* img_conv3, const uint8_t* frames, int n, float* a1, float* a2, float* a3) {
  int launches = 0;
  return pl.C == 1 ? conv_forward_tf32<1>(s, pl, P, img_conv2, img_conv3, frames, n, 1, a1, a2, a3, 2, false, nullptr,
                                          &launches)
                   : conv_forward_tf32<4>(s, pl, P, img_conv2, img_conv3, frames, n, 1, a1, a2, a3, 2, false, nullptr,
                                          &launches);
}

int policy_conv_images_tf32(cudaStream_t s, const TrunkLayout& pl, const float* P, uint8_t* img_conv2,
                            uint8_t* img_conv3) {
  return conv_images_tf32(s, pl, P, img_conv2, img_conv3);
}

// The recurrence at the handle's width: the one-CTA-per-sequence kernels at L = 64, a cluster kernel otherwise, with
// as many clusters as there are R-sequence chunks, up to what the device places at once (drl_r2d2_create checks >= 1).
template <int L>
static cudaError_t lstm_fwd_cluster(cudaStream_t s, int max_clusters, const float* zx, const float* bias, const float* Wh,
                                    const R2In& in, const R2Acts& act, float* c_last, int B, int S) {
  using K = R2Clu<L>;
  const int ncl = std::min(cdiv(B, K::R), max_clusters);
  return launch_cluster_k(r2d2_lstm_fwd_cluster_kernel<L>, K::CL, ncl * K::CL, K::T, K::kFwdSmem, s, zx, bias, Wh, in.h0,
                          in.c0, in.done, act.gates, act.tc, act.hout, act.hin, act.cin, c_last, B, S);
}
static cudaError_t lstm_fwd(cudaStream_t s, const drl_r2d2* h, const float* bias, const float* Wh, const R2In& in,
                            const R2Acts& act, float* c_last, int B, int S) {
  if (h->L == 256) return lstm_fwd_cluster<256>(s, h->clusters_fwd, act.zx, bias, Wh, in, act, c_last, B, S);
  if (h->L == 512) return lstm_fwd_cluster<512>(s, h->clusters_fwd, act.zx, bias, Wh, in, act, c_last, B, S);
  return launch_k(r2d2_lstm_fwd_kernel, B, kR2G, kR2FwdSmem, s, act.zx, 1, (size_t)0, bias, Wh, in.h0, in.c0, in.done,
                  act.gates, act.tc, act.hout, act.hin, act.cin, c_last, B, S);
}
template <int L>
static cudaError_t lstm_bwd_cluster(cudaStream_t s, int max_clusters, const R2Bwd& bw, const R2Acts& act, const float* Wh,
                                    const uint8_t* done, int B, int S) {
  using K = R2Clu<L>;
  const int ncl = std::min(cdiv(B, K::R), max_clusters);
  return launch_cluster_k(r2d2_lstm_bwd_cluster_kernel<L>, K::CL, ncl * K::CL, K::T, K::kBwdSmem, s, bw.dhout, act.gates,
                          act.tc, act.cin, Wh, done, bw.dz, B, S);
}
static cudaError_t lstm_bwd(cudaStream_t s, const drl_r2d2* h, const R2Bwd& bw, const R2Acts& act, const float* Wh,
                            const uint8_t* done, int B, int S) {
  if (h->L == 256) return lstm_bwd_cluster<256>(s, h->clusters_bwd, bw, act, Wh, done, B, S);
  if (h->L == 512) return lstm_bwd_cluster<512>(s, h->clusters_bwd, bw, act, Wh, done, B, S);
  return launch_k(r2d2_lstm_bwd_kernel, B, kR2G, kR2BwdSmem, s, bw.dhout, act.gates, act.tc, act.cin, Wh, done, bw.dz, B,
                  S);
}

// Forward of one scope over B sequences of S steps (rows m = t*B + b).  c_last (optional): un-masked c_t (act path).
static int r2_forward(const drl_r2d2* h, const Streams& st, const float* P, const WeightImages& wi, const R2In& in,
                      const R2Acts& act, float* c_last, int B, int S, int mode, bool retile_fwd, bool retile_bwd, bool tgt,
                      int* launches) {
  const R2Layout& pl = h->pl;
  const int L = h->L, G = 4 * h->L;
  const int M = B * S;
  const RowMap map{B, S};
  int n = 0;
  cudaStream_t s = st.main;
  const cudaStream_t side = st.par ? st.side : st.main;
  DRL_TRY(fork_to_side(st, 0));
  s = side;
  if (retile_fwd && mode >= 2) {
    prof_mark(s, tgt ? "target_weight_retile" : "weight_retile");
    DRL_TRY(conv_images_tf32(s, pl, P, wi.img[1], wi.img[2]));
    n += 2;
  }
  if (st.par) DRL_CUDA_CHECK(cudaEventRecord(st.ev[7], side));
  KERNEL(tgt ? "target_emb_fwd" : "emb_fwd",
         emb_forward(s, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, act.e1, act.table, pl.A), 1);
  if (retile_bwd && mode >= 2) {
    prof_mark(s, "weight_retile_bwd");
    DRL_TRY(conv_dcol_images_tf32(s, pl, P, wi.img[5], wi.img[6]));
    n += 2;
  }
  s = st.main;
  const cudaEvent_t images_ready = st.par ? st.ev[7] : nullptr;
  DRL_TRY(pl.C == 1 ? conv_forward_tf32<1>(s, pl, P, wi.img[1], wi.img[2], in.frames, B, S, act.a1, act.a2, act.a3,
                                           mode, tgt, images_ready, &n)
                    : conv_forward_tf32<4>(s, pl, P, wi.img[1], wi.img[2], in.frames, B, S, act.a1, act.a2, act.a3,
                                           mode, tgt, images_ready, &n));
  DRL_TRY(join_from_side(st, 1));
  // input half of the LSTM contraction for all S steps at once: [M, 3392] x W[:3392, :4L] (split-K partial sums)
  const SplitPlan sp = plan_r2_x(M, mode, G);
  {
    R2XA al{act.a3, act.table, in.pa, map};
    PlainB bl{P + pl.lstm_w, G, 0};
    EpRaw<false> ep{act.zpart, G, (size_t)M * G, 1.0f, 0, G};
    GEMM(tgt ? "target_lstm_x_fwd" : "lstm_x_fwd", CfgMid, U256, al, bl, ep, M, G, kR2Cat, sp.splits, sp.kchunk, sp.kchunk);
  }
  KERNEL(tgt ? "target_lstm_x_reduce" : "lstm_x_reduce",
         splitk_reduce(s, act.zpart, (size_t)M * G, sp.splits, act.zx, (size_t)M * G), 1);
  prof_mark(s, tgt ? "target_lstm_unroll_fwd" : "lstm_unroll_fwd");
  DRL_CUDA_CHECK(lstm_fwd(s, h, P + pl.lstm_b, P + pl.lstm_w + (size_t)kR2Cat * G, in, act, c_last, B, S));
  ++n;
  {  // dense 128 ReLU (model/r2d2_lstm.py:50)
    PlainA al{act.hout, L, 0};
    PlainB bl{P + pl.q1_w, kR2H, 0};
    EpBiasAct<true, true> ep{act.q1, kR2H, 0, P + pl.q1_b, 0, 1.0f};
    GEMM_FFMA(tgt ? "target_q1_fwd" : "q1_fwd", CfgSmall, al, bl, ep, M, kR2H, L, 1, L, 0);
  }
  prof_mark(s, tgt ? "target_q_out_fwd" : "q_out_fwd");
  DRL_CUDA_CHECK((launch_k(r2d2_out_kernel, cdiv(M, 4), 128, 0, s, act.q1, P + pl.value_w, P + pl.value_b, P + pl.mean_w,
                           P + pl.mean_b, act.q, M, pl.A)));
  ++n;
  if (launches) *launches += n;
  return DRL_OK;
}

static int r2_backward(const drl_r2d2* h, const Streams& st, const float* P, const WeightImages& wi, float* G,
                       const R2In& in, const R2Acts& act, const R2Bwd& bw, int B, int S, int mode, int* launches) {
  const R2Layout& pl = h->pl;
  const int L = h->L, NG = 4 * h->L;
  const int M = B * S;
  const RowMap map{B, S};
  cudaStream_t s = st.main;
  const cudaStream_t side = st.par ? st.side : st.main;
  const int A = pl.A;
  int n = 0;
  prof_mark(s, "q_out_bwd");
  DRL_CUDA_CHECK((launch_k(r2d2_out_bwd_kernel, M, kR2H, 0, s, bw.dq, bw.dmean, P + pl.value_w, P + pl.mean_w, act.q1,
                           bw.dq1, A)));
  ++n;
  DRL_TRY(fork_to_side(st, 0));
  s = side;
  {  // d value [128(+1), A]
    PlainAT al{act.q1, kR2H, 0};
    PlainB bl{bw.dq, 32, 0};
    EpRaw<true> ep{G + pl.value_w, A, 0, 1.0f, kR2H, A};
    GEMM_FFMA("value_wgrad", CfgSmall, al, bl, ep, kR2H, 32, M, 1, M, 0);
  }
  {  // d mean [128(+1), 1]
    PlainAT al{act.q1, kR2H, 0};
    PlainB bl{bw.dmean, 32, 0};
    EpRaw<true> ep{G + pl.mean_w, 1, 0, 1.0f, kR2H, 1};
    GEMM_FFMA("mean_wgrad", CfgSmall, al, bl, ep, kR2H, 32, M, 1, M, 0);
  }
  {  // d q1 kernel [L(+1), 128] = hout^T dq1
    PlainAT al{act.hout, L, 0};
    PlainB bl{bw.dq1, kR2H, 0};
    EpRaw<true> ep{G + pl.q1_w, kR2H, 0, 1.0f, L, kR2H};
    GEMM_FFMA("q1_wgrad", CfgSmall, al, bl, ep, L, kR2H, M, 1, M, 0);
  }
  s = st.main;
  {  // dhout = dq1 W1^T
    PlainA al{bw.dq1, kR2H, 0};
    PlainBT bl{P + pl.q1_w, kR2H, 0};
    EpRaw<false> ep{bw.dhout, L, 0, 1.0f, 0, L};
    GEMM_FFMA("q1_dgrad", CfgSmall, al, bl, ep, M, L, kR2H, 1, kR2H, 0);
  }
  prof_mark(s, "lstm_unroll_bwd");
  DRL_CUDA_CHECK(lstm_bwd(s, h, bw, act, P + pl.lstm_w + (size_t)kR2Cat * NG, in.done, B, S));
  ++n;
  DRL_TRY(fork_to_side(st, 3));
  s = side;
  {  // d lstm kernel [3392 + L (+1), 4L] = [x | h_in]^T dz ; bias gradient = column sums of dz
    LstmHinAT al{act.a3, act.table, in.pa, act.hin, map, L};
    PlainB bl{bw.dz, NG, 0};
    EpRaw<true> ep{G + pl.lstm_w, NG, 0, 1.0f, kR2Cat + L, NG};
    GEMM("lstm_wgrad", CfgBig, U256, al, bl, ep, kR2Cat + L, NG, M, 1, M, 0);
  }
  s = st.main;
  {  // d[a3 | emb] = dz W[:3392]^T
    PlainA al{bw.dz, NG, 0};
    PlainBT bl{P + pl.lstm_w, NG, 0};
    EpLstmDx ep{bw.da3, act.a3, bw.du};
    GEMM("lstm_dgrad", CfgMid, U128, al, bl, ep, M, kR2Cat, NG, 1, NG, 0);
  }
  DRL_TRY(fork_to_side(st, 4));
  s = side;
  KERNEL("emb_bwd",
         emb_backward(s, bw.du, in.pa, act.e1, act.table, P + pl.emb2_w, bw.dpre2, bw.dpre1, G + pl.emb1_w,
                      G + pl.emb1_b, G + pl.emb2_w, G + pl.emb2_b, bw.wg_part, M, B, S, A), 4);
  DRL_TRY(pl.C == 1 ? conv_backward_tf32<1>(st, pl, P, wi, G, in.frames, map, M, act, bw, mode, &n)
                    : conv_backward_tf32<4>(st, pl, P, wi, G, in.frames, map, M, act, bw, mode, &n));
  DRL_TRY(join_from_side(st, 6));
  if (launches) *launches += n;
  return DRL_OK;
}

}  // namespace drl

using namespace drl;

// both unrolls + TD kernel over nb sequences held by `in` (r2d2_defs.cuh)
int drl::enqueue_forward_td(drl_r2d2* h, const R2In& in, int nb, bool train, float* td_host, int* launches) {
  const Streams st = h->streams(), tst = h->target_streams();
  // the two unrolls are independent (and each recurrence kernel only occupies nb SMs): the target scope runs on its
  // own stream pair beside the main scope and joins before the TD kernel
  if (h->par) {
    DRL_CUDA_CHECK(cudaEventRecord(h->ev_tfork, h->compute));
    DRL_CUDA_CHECK(cudaStreamWaitEvent(h->tmain, h->ev_tfork, 0));
  }
  DRL_TRY(r2_forward(h, tst, h->target, h->twi, in, h->tact, nullptr, nb, h->S, h->mode, h->target_images_stale, false,
                     true, launches));
  h->target_images_stale = false;
  if (h->par) DRL_CUDA_CHECK(cudaEventRecord(h->ev_tjoin, h->tmain));
  DRL_TRY(r2_forward(h, st, h->params, h->wi, in, h->act, nullptr, nb, h->S, h->mode, h->images_stale,
                     h->images_stale, false, launches));
  h->images_stale = false;
  if (h->par) DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, h->ev_tjoin, 0));
  R2TdArgs a{};
  a.mq = h->act.q; a.tq = h->tact.q;
  a.action = in.action; a.reward = in.reward; a.done = in.done; a.weight = train ? in.weight : nullptr;
  a.discount = h->cfg.discount_factor; a.B = nb; a.S = h->S; a.burn_in = h->cfg.burn_in; a.A = h->A;
  a.sav = h->sav; a.target_value = h->target_value; a.td_dev = h->td_dev; a.td_host = td_host;
  a.dq = train ? h->bwd.dq : nullptr; a.dmean = train ? h->bwd.dmean : nullptr;
  a.loss = train ? h->loss : nullptr;
  prof_mark(h->compute, "td_target_loss");
  const int n_step = std::max(h->cfg.n_step, 1);
  if (n_step > 1 || h->cfg.priority_rule == 1)
    DRL_CUDA_CHECK((launch_k(r2d2_td_nstep_kernel, 1, 256, 0, h->compute, a, n_step, h->cfg.priority_rule,
                             h->cfg.priority_eta)));
  else
    DRL_CUDA_CHECK((launch_k(r2d2_td_kernel, 1, 256, 0, h->compute, a)));
  if (launches) *launches += 1;
  return DRL_OK;
}

namespace {

constexpr const char* kName = "r2d2";

int alloc_acts(drl_r2d2* h, R2Acts& a) {
  const size_t M = (size_t)h->B * h->S, A = h->A, L = h->L, G = 4 * L;
  DRL_TRY(alloc_trunk_acts(h, a, M, A));
  size_t zmax = 0;
  for (int mode = 1; mode <= 2; ++mode)
    for (int m = 1; m <= (int)M; ++m) zmax = std::max(zmax, (size_t)plan_r2_x(m, mode, (int)G).splits * m * G);
  DRL_TRY(dev_alloc(h, &a.zpart, zmax));
  DRL_TRY(dev_alloc(h, &a.zx, M * G));
  DRL_TRY(dev_alloc(h, &a.gates, M * G));
  DRL_TRY(dev_alloc(h, &a.tc, M * L));
  DRL_TRY(dev_alloc(h, &a.hout, M * L));
  DRL_TRY(dev_alloc(h, &a.hin, M * L));
  DRL_TRY(dev_alloc(h, &a.cin, M * L));
  DRL_TRY(dev_alloc(h, &a.q1, M * kR2H));
  DRL_TRY(dev_alloc(h, &a.q, M * A));
  return DRL_OK;
}

int fwd_bwd(LearnerCore* core, int slot, int* launches) {
  drl_r2d2* h = static_cast<drl_r2d2*>(core);
  const R2In& in = h->in[slot];
  DRL_TRY(enqueue_forward_td(h, in, h->B, true, h->d_td + (size_t)slot * h->B, launches));
  return r2_backward(h, h->streams(), h->params, h->wi, h->grads, in, h->act, h->bwd, h->B, h->S, h->mode, launches);
}

// H2D of nb sequences into slot s on `stream` (fields that are null are skipped)
int stage_into(drl_r2d2* h, const R2In& s, cudaStream_t stream, int nb, int steps, const uint8_t* state,
               const int32_t* previous_action, const int32_t* action, const float* h0, const float* c0, const float* reward,
               const uint8_t* done, const float* weight) {
  auto cp = [&](const void* dst, const void* src, size_t bytes) -> cudaError_t {
    return cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, stream);
  };
  const size_t n = (size_t)nb * steps;
  DRL_CUDA_CHECK(cp(s.frames, state, n * h->frame));
  DRL_CUDA_CHECK(cp(s.pa, previous_action, n * 4));
  if (action) DRL_CUDA_CHECK(cp(s.action, action, n * 4));
  DRL_CUDA_CHECK(cp(s.h0, h0, (size_t)nb * h->L * 4));
  DRL_CUDA_CHECK(cp(s.c0, c0, (size_t)nb * h->L * 4));
  if (reward) DRL_CUDA_CHECK(cp(s.reward, reward, n * 4));
  if (done) DRL_CUDA_CHECK(cp(s.done, done, n));
  if (reward) DRL_CUDA_CHECK(cp(s.weight, weight ? weight : h->h_ones, (size_t)nb * 4));
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_r2d2_create(const drl_r2d2_config* cfg, drl_r2d2** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || (cfg->channels != 1 && cfg->channels != 4)) {
    set_error("only 84x84x1 (config.json:91) and 84x84x4 frames are supported (got %dx%dx%d)", cfg->height, cfg->width, cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->lstm_size != kR2L && cfg->lstm_size != 256 && cfg->lstm_size != 512) {
    set_error("lstm_size must be 64 (config.json:93), 256 or 512 (got %d)", cfg->lstm_size);
    return DRL_ERR_INVALID;
  }
  if (cfg->num_action < 2 || cfg->num_action > 32) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  if (cfg->batch < 1) { set_error("batch must be >= 1"); return DRL_ERR_INVALID; }
  if (cfg->seq_len < 2 || cfg->burn_in < 0 || cfg->burn_in > cfg->seq_len - 2) {
    set_error("need seq_len >= 2 and 0 <= burn_in <= seq_len - 2 (got seq_len %d, burn_in %d)", cfg->seq_len, cfg->burn_in);
    return DRL_ERR_INVALID;
  }
  if (cfg->math_mode < 0 || cfg->math_mode > 2) { set_error("math_mode must be 0 (default), 1 (FP32 FFMA) or 2 (wgmma 3xTF32)"); return DRL_ERR_INVALID; }
  const int Nt = cfg->seq_len - cfg->burn_in - 1;
  if (cfg->n_step < 0 || cfg->n_step > Nt) {
    set_error("n_step must be 0 or 1 (one-step targets) or at most seq_len - burn_in - 1 = %d (got %d)", Nt, cfg->n_step);
    return DRL_ERR_INVALID;
  }
  if (cfg->priority_rule != 0 && cfg->priority_rule != 1) {
    set_error("priority_rule must be 0 (|mean td|) or 1 (eta max |td| + (1 - eta) mean |td|) (got %d)", cfg->priority_rule);
    return DRL_ERR_INVALID;
  }
  if (cfg->priority_rule == 1 && !(cfg->priority_eta >= 0.0f && cfg->priority_eta <= 1.0f)) {
    set_error("priority_eta must be finite and in [0, 1] (got %g)", (double)cfg->priority_eta);
    return DRL_ERR_INVALID;
  }
  if (drl_device_count() <= cfg->device) { set_error("CUDA device %d not available (no CPU fallback)", cfg->device); return DRL_ERR_CUDA; }
  drl_r2d2* h = new drl_r2d2();
  h->cfg = *cfg;
  h->device = cfg->device;
  h->num_slots = cfg->num_slots < 1 ? 2 : cfg->num_slots;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->mode = (cfg->math_mode == 0) ? DRL_DEFAULT_MATH_MODE : cfg->math_mode;
  h->B = cfg->batch; h->S = cfg->seq_len; h->A = cfg->num_action; h->C = cfg->channels; h->L = cfg->lstm_size;
  h->Nt = cfg->seq_len - cfg->burn_in - 1;
  h->frame = (size_t)Geo::IH * Geo::IW * h->C;
  h->pl.init(h->A, h->C, h->L);
  h->layout = &h->pl;
  h->fwd_bwd = fwd_bwd;
  AdamState& o = h->opt;
  o.start_lr = cfg->learning_rate; o.end_lr = cfg->learning_rate; o.learning_frame = 1.0;   // constant (agent/r2d2.py:91)
  o.clip_norm = 0.0f;                                                                        // minimize(): no clipping
  int rc = [&]() -> int {
    const size_t B = h->B, S = h->S, M = B * S, A = h->A, L = h->L;
    size_t off = 0;
    const size_t o_fr = off; off = align_up(off + M * h->frame, 256);
    const size_t o_pa = off; off = align_up(off + M * 4, 256);
    const size_t o_ac = off; off = align_up(off + M * 4, 256);
    const size_t o_h = off; off = align_up(off + M * L * 4, 256);    // room for M rows: the act path stages n <= M states
    const size_t o_c = off; off = align_up(off + M * L * 4, 256);
    const size_t o_rw = off; off = align_up(off + M * 4, 256);
    const size_t o_dn = off; off = align_up(off + M, 256);
    const size_t o_wt = off; off = align_up(off + M * 4, 256);
    DRL_TRY(adam_learner_init(h, off, M));
    if (L == 256) DRL_TRY(r2d2_cluster_setup<256>(&h->clusters_fwd, &h->clusters_bwd));
    if (L == 512) DRL_TRY(r2d2_cluster_setup<512>(&h->clusters_fwd, &h->clusters_bwd));
    for (const LearnerSlot& s : h->slots)
      h->in.push_back(R2In{s.base + o_fr, reinterpret_cast<int32_t*>(s.base + o_pa),
                           reinterpret_cast<int32_t*>(s.base + o_ac), reinterpret_cast<float*>(s.base + o_h),
                           reinterpret_cast<float*>(s.base + o_c), reinterpret_cast<float*>(s.base + o_rw),
                           s.base + o_dn, reinterpret_cast<float*>(s.base + o_wt)});
    DRL_TRY(alloc_acts(h, h->act));
    DRL_TRY(alloc_acts(h, h->tact));
    R2Bwd& b = h->bwd;
    DRL_TRY(dev_alloc(h, &b.dq, M * 32));
    DRL_TRY(dev_alloc(h, &b.dmean, M * 32));
    DRL_TRY(dev_alloc(h, &b.dq1, M * kR2H));
    DRL_TRY(dev_alloc(h, &b.dhout, M * L));
    DRL_TRY(dev_alloc(h, &b.dz, M * 4 * L));
    DRL_TRY(alloc_trunk_bwd(h, b, M, A, h->C, true));
    const size_t Nt = h->Nt;
    DRL_TRY(dev_alloc(h, &h->sav, B * Nt));
    DRL_TRY(dev_alloc(h, &h->target_value, B * Nt));
    DRL_TRY(dev_alloc(h, &h->td_dev, B));
    DRL_TRY(dev_alloc(h, &h->c_last, M * L));
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_r2d2_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_r2d2_destroy(drl_r2d2* h) {
  if (!h) return DRL_OK;
  adam_learner_release(h);
  delete h;
  return DRL_OK;
}

int drl_r2d2_param_count(const drl_r2d2* h, int64_t* n) { return learner_param_count(h, kName, n); }
int drl_r2d2_set_params(drl_r2d2* h, int32_t which, const float* host_flat, int64_t n) {
  return adam_set_params(h, kName, which, host_flat, n);
}
int drl_r2d2_get_params(drl_r2d2* h, int32_t which, float* host_flat, int64_t n) {
  return adam_get_params(h, kName, which, host_flat, n);
}
int drl_r2d2_set_opt_state(drl_r2d2* h, const float* host_m, const float* host_v, int64_t n, int64_t step,
                           float beta1_power, float beta2_power) {
  return adam_set_opt_state(h, kName, host_m, host_v, n, step, beta1_power, beta2_power);
}
int drl_r2d2_get_opt_state(drl_r2d2* h, float* host_m, float* host_v, int64_t n, int64_t* step, float* beta1_power,
                           float* beta2_power) {
  return adam_get_opt_state(h, kName, host_m, host_v, n, step, beta1_power, beta2_power);
}
int drl_r2d2_get_grads(drl_r2d2* h, float* host_flat, int64_t n) { return learner_get_grads(h, kName, h->grads, host_flat, n); }
int drl_r2d2_main_to_target(drl_r2d2* h) { return adam_main_to_target(h, kName); }

int drl_r2d2_stage(drl_r2d2* h, int32_t slot, const uint8_t* state, const int32_t* previous_action, const int32_t* action,
                   const float* h0, const float* c0, const float* reward, const uint8_t* done, const float* weight) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  if (!state || !previous_action || !action || !h0 || !c0 || !reward || !done) { set_error("stage: null input pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  LearnerSlot& s = h->slots[slot];
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, s.consumed, 0));
  DRL_TRY(stage_into(h, h->in[slot], h->copy, h->B, h->S, state, previous_action, action, h0, c0, reward, done, weight));
  DRL_CUDA_CHECK(cudaEventRecord(s.staged, h->copy));
  s.has_data = true;
  return DRL_OK;
}

}  // extern "C"

int drl::r2d2_params_snapshot(drl_r2d2* h, int device, int num_action, int channels, cudaStream_t dst_stream,
                              float* dst, cudaEvent_t ev_ready, cudaEvent_t ev_copied) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->A != num_action || h->C != channels) {
    set_error("sync: the learner has num_action %d and %d channels, the policy %d and %d", h->A, h->C, num_action,
              channels);
    return DRL_ERR_INVALID;
  }
  if (h->L != kR2L) {
    set_error("sync: the learner has lstm_size %d, the policy engine %d", h->L, kR2L);
    return DRL_ERR_INVALID;
  }
  return learner_params_snapshot(h, kName, device, dst_stream, dst, ev_ready, ev_copied);
}

extern "C" {

int drl_r2d2_step_async(drl_r2d2* h, int32_t slot) { return learner_step_async(h, kName, slot); }
int drl_r2d2_forward_backward(drl_r2d2* h, int32_t slot) { return learner_forward_backward(h, kName, slot); }
int drl_r2d2_grad_bucket(drl_r2d2* h, void** dev_ptr, int64_t* count) { return learner_grad_bucket(h, kName, dev_ptr, count); }
int drl_r2d2_apply(drl_r2d2* h, float grad_scale) { return learner_apply(h, kName, grad_scale); }

int drl_r2d2_wait(drl_r2d2* h, drl_r2d2_out* out, float* td_error) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);     // the scalar row stays valid while it is read
  const float* r = nullptr;
  DRL_TRY(adam_wait(h, kName, &r, td_error));
  if (out) {
    out->loss = r[0];
    out->grad_norm = r[2];
    out->step = step_of(r);
  }
  return DRL_OK;
}
int drl_r2d2_step(drl_r2d2* h, int32_t slot, drl_r2d2_out* out, float* td_error) {
  DRL_TRY(drl_r2d2_step_async(h, slot));
  return drl_r2d2_wait(h, out, td_error);
}

int drl_r2d2_td_error(drl_r2d2* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const int32_t* action,
                      const float* h0, const float* c0, const float* reward, const uint8_t* done, float* td_error) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > h->B) { set_error("td_error: n must be in [1, %d]", h->B); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !action || !h0 || !c0 || !reward || !done || !td_error) { set_error("td_error: null pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  const R2In& s = h->in[h->num_slots];
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  DRL_TRY(stage_into(h, s, h->compute, n, h->S, state, previous_action, action, h0, c0, reward, done, nullptr));
  DRL_TRY(enqueue_forward_td(h, s, n, false, nullptr, nullptr));
  DRL_CUDA_CHECK(cudaMemcpyAsync(td_error, h->td_dev, (size_t)n * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  h->last_n = n;
  return DRL_OK;
}

int drl_r2d2_act(drl_r2d2* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
                 const float* c_in, float* q_value, float* h_out, float* c_out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int M = h->B * h->S;
  if (n < 1 || n > M) { set_error("act: n must be in [1, %d]", M); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !h_in || !c_in) { set_error("act: null pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  R2In in = h->in[h->num_slots];
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  DRL_TRY(stage_into(h, in, h->compute, n, 1, state, previous_action, nullptr, h_in, c_in, nullptr, nullptr, nullptr));
  in.done = nullptr;                                     // a single step: nothing is carried
  DRL_TRY(r2_forward(h, h->streams(), h->params, h->wi, in, h->act, h->c_last, n, 1, h->mode, h->images_stale,
                     h->images_stale, false, nullptr));
  h->images_stale = false;
  if (q_value) DRL_CUDA_CHECK(cudaMemcpyAsync(q_value, h->act.q, (size_t)n * h->A * 4, cudaMemcpyDeviceToHost, h->compute));
  if (h_out) DRL_CUDA_CHECK(cudaMemcpyAsync(h_out, h->act.hout, (size_t)n * h->L * 4, cudaMemcpyDeviceToHost, h->compute));
  if (c_out) DRL_CUDA_CHECK(cudaMemcpyAsync(c_out, h->c_last, (size_t)n * h->L * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  h->last_n = 0;
  return DRL_OK;
}

int drl_r2d2_taps(drl_r2d2* h, float* main_q, float* target_q, float* target_value, float* state_action_value) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  if (h->last_n < 1) { set_error("taps: no step or td_error call has run"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  const int nb = h->last_n, S = h->S, A = h->A;
  // time-major device rows -> batch-major host arrays [nb, S, A]
  for (int which = 0; which < 2; ++which) {
    float* dst = which == 0 ? main_q : target_q;
    if (!dst) continue;
    std::vector<float> tmp((size_t)nb * S * A);
    DRL_CUDA_CHECK(cudaMemcpy(tmp.data(), which == 0 ? h->act.q : h->tact.q, tmp.size() * 4, cudaMemcpyDeviceToHost));
    for (int t = 0; t < S; ++t)
      for (int b = 0; b < nb; ++b)
        memcpy(dst + ((size_t)b * S + t) * A, tmp.data() + ((size_t)t * nb + b) * A, A * sizeof(float));
  }
  const size_t nt = (size_t)nb * h->Nt;
  if (target_value) DRL_CUDA_CHECK(cudaMemcpy(target_value, h->target_value, nt * 4, cudaMemcpyDeviceToHost));
  if (state_action_value) DRL_CUDA_CHECK(cudaMemcpy(state_action_value, h->sav, nt * 4, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_r2d2_read_buffer(drl_r2d2* h, const char* name, float* host_dst, int64_t n) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!name || !host_dst) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  if (h->last_n < 1) { set_error("read_buffer: no step or td_error call has run"); return DRL_ERR_STATE; }
  const size_t M = (size_t)h->last_n * h->S, A = h->A, L = h->L;
  const NamedBuffer tab[] = {
      {"a1", h->act.a1, M * 400 * 32}, {"a2", h->act.a2, M * 81 * 64}, {"a3", h->act.a3, M * Geo::FLAT},
      {"emb", h->act.table, A * Geo::EMB}, {"e1", h->act.e1, A * Geo::EMB}, {"q1", h->act.q1, M * kR2H},
      {"hout", h->act.hout, M * L}, {"hin", h->act.hin, M * L}, {"cin", h->act.cin, M * L},
      {"gates", h->act.gates, M * 4 * L}, {"dz", h->bwd.dz, M * 4 * L}, {"dhout", h->bwd.dhout, M * L},
      {"zx", h->act.zx, M * 4 * L}, {"tc", h->act.tc, M * L}, {"q", h->act.q, M * A},
      {"dq", h->bwd.dq, M * 32}, {"dmean", h->bwd.dmean, M * 32}, {"dq1", h->bwd.dq1, M * kR2H},
      {"du", h->bwd.du, M * Geo::EMB}, {"da3", h->bwd.da3, M * Geo::FLAT}, {"da2", h->bwd.da2, M * 81 * 64},
      {"da1", h->bwd.da1, M * 400 * 32}};
  return read_named_buffer(h, tab, sizeof(tab) / sizeof(tab[0]), name, host_dst, n);
}

// The launch plan of an R2D2 step over B sequences of S steps of C-channel frames in math mode `mode` at width
// `lstm_size` (M = B*S rows, all of which receive gradient), read by the per-kernel tests to assert which edges a case
// reaches: out[0] = split-K count of lstm_x_fwd (N = 4 lstm_size), out[1..3] = split-K count of the conv1 / conv2 /
// conv3 weight gradients (conv1: the single-channel plan when C == 1), out[4] = sequences per cluster pass of the
// recurrence (R2Clu<L>::R; 0 at 64, which runs one CTA per sequence).
int drl_debug_r2d2_launch_plan(int32_t B, int32_t S, int32_t C, int32_t mode, int32_t lstm_size, int32_t* out) {
  if (!out || B < 1 || S < 1 || (C != 1 && C != 4) || mode < 1 || mode > 2 ||
      (lstm_size != kR2L && lstm_size != 256 && lstm_size != 512)) {
    set_error("r2d2_launch_plan: need out, B >= 1, S >= 1, C 1 or 4, mode 1 or 2, lstm_size 64, 256 or 512");
    return DRL_ERR_INVALID;
  }
  const int M = B * S;
  out[0] = plan_r2_x(M, mode, 4 * lstm_size).splits;
  out[1] = C == 1 ? plan_conv1_wgrad_c1(M).splits : plan_conv1_wgrad(M, mode).splits;
  out[2] = plan_conv2_wgrad(M, mode).splits;
  out[3] = plan_conv3_wgrad(M, mode).splits;
  out[4] = lstm_size == 256 ? R2Clu<256>::R : lstm_size == 512 ? R2Clu<512>::R : 0;
  return DRL_OK;
}

int drl_r2d2_profile_step(drl_r2d2* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels,
                          int32_t* count) {
  return learner_profile_step(h, kName, slot, names, names_len, ms, max_kernels, count);
}
int drl_r2d2_last_step_ms(drl_r2d2* h, float* ms) { return learner_last_step_ms(h, kName, ms); }
int drl_r2d2_stream(drl_r2d2* h, void** stream) { return learner_stream(h, kName, stream); }
int drl_r2d2_launches_per_step(const drl_r2d2* h, int32_t* n) { return learner_launches_per_step(h, kName, n); }

int drl_r2d2_recurrence_clusters(const drl_r2d2* h, int32_t* cluster_size, int32_t* max_fwd, int32_t* max_bwd) {
  DRL_TRY(check_handle(h, kName));
  if (!cluster_size || !max_fwd || !max_bwd) { set_error("null argument"); return DRL_ERR_INVALID; }
  *cluster_size = h->L == kR2L ? 0 : h->L / 32;
  *max_fwd = h->clusters_fwd;
  *max_bwd = h->clusters_bwd;
  return DRL_OK;
}

}  // extern "C"
