// apex.cu -- the Ape-X DQN learner behind drl_apex_* (include/drl_b200.h): replaces apex.Agent's learner graph
// (agent/apex.py:12-76) over the dueling network of model/apex_value.py:4-66, optimizer/dqn.py:3-7 and TF1 Adam.
//
// The reference builds three network copies -- main(s, prev_a), main(s', a), target(s', a) (model/apex_value.py:43-66).
// Here the two main-network evaluations are ONE forward over 2B rows [s ; s'] (the B rows that receive gradient are
// the contiguous prefix, exactly like the B*(T-2) prefix of the IMPALA learner), the target network is one forward
// over the B rows s'.  The attention_CNN and the action embedding are the same layers as IMPALA's, so they run
// through the same gather-GEMM kernels (layer_defs.cuh); the two streams of the dueling head share their input
// concat = [a3 | emb(prev_a)] (K = 3392), so their first layers are one split-K GEMM with N = 2 x 256.
#include <string.h>

#include <string>
#include <vector>

#include "adam_learner.cuh"
#include "apex_defs.cuh"
#include "layer_defs.cuh"
#include "traj_queue.cuh"

namespace drl {

static SplitPlan plan_head1(int M) { return plan_split(kCat, cdiv(M, CfgMid::BM) * (kHeadN / CfgMid::BN), 16, 1); }

// hid1[z][m][j] = relu(sum_s zpart[s][m][z*256 + j] + b1[z][j])   (first layers of both streams, model/apex_value.py:17-19)
__global__ void __launch_bounds__(256) apex_hid1_kernel(const float* __restrict__ zpart, int nsplit, size_t slab,
                                                         const float* __restrict__ bv, const float* __restrict__ bm,
                                                         float* __restrict__ hid1, int M) {
  kernel_prologue();
  const int m = blockIdx.x, j = threadIdx.x;
#pragma unroll
  for (int z = 0; z < 2; ++z) {
    float acc = 0.f;
    for (int s = 0; s < nsplit; ++s) acc += zpart[(size_t)s * slab + (size_t)m * kHeadN + z * Geo::HID + j];
    acc += (z == 0 ? bv[j] : bm[j]);
    hid1[((size_t)z * M + m) * Geo::HID + j] = fmaxf(acc, 0.f);
  }
}

// ------------------------------------------------------------------------------------------
// TD target, loss and head gradients (agent/apex.py:43-65, optimizer/dqn.py:3-7), one thread per transition b:
//   q_main(b)      = vstream[b] - mstream[b]                         (model/apex_value.py:40)
//   next_action    = argmax_a q_main(n + b)  (first maximum)          rows n.. hold main(s', a)
//   target_value   = q_target(b)[next_action] * gamma * (1 - done) + clip(r)     (stop_gradient)
//   sav            = q_main(b)[action]
//   loss           = mean_b w_b (target_value - sav)^2
//   d loss / d vstream[b][a] = -2 w_b (target - sav) / n for a == action ; d loss / d mstream[b] = the negative of it
// One block: the loss is a fixed-order block reduction (deterministic).
// ------------------------------------------------------------------------------------------
struct TdArgs {
  const float* vstream; const float* mstream;     // main network, 2n rows
  const float* tvstream; const float* tmstream;   // target network, n rows (s')
  const int32_t* action; const float* reward; const uint8_t* done; const float* weight;   // weight may be null (= 1)
  float discount; int clip; int n; int A;
  float* main_q; float* next_main_q; float* target_q;   // [n, A] taps
  float* target_value; float* sav;                      // [n]
  float* td_dev; float* td_host;                        // [n] |target - sav| (device copy, mapped pinned copy or null)
  float* dq; float* dmean;                              // [n, 32] or null (forward-only call)
  float* loss;                                          // [1] or null
};

__global__ void __launch_bounds__(256) apex_td_kernel(TdArgs a) {
  kernel_prologue();
  __shared__ float red[8];
  float part = 0.f;
  for (int b = threadIdx.x; b < a.n; b += blockDim.x) {
    const float mm = a.mstream[b], mn = a.mstream[a.n + b], mt = a.tmstream[b];
    const int act = a.action[b];
    float best = -INFINITY, sav = 0.f;
    int arg = 0;
    for (int k = 0; k < a.A; ++k) {
      const float qm = a.vstream[(size_t)b * a.A + k] - mm;
      const float qn = a.vstream[(size_t)(a.n + b) * a.A + k] - mn;
      const float qt = a.tvstream[(size_t)b * a.A + k] - mt;
      a.main_q[(size_t)b * a.A + k] = qm;
      a.next_main_q[(size_t)b * a.A + k] = qn;
      a.target_q[(size_t)b * a.A + k] = qt;
      if (k == act) sav = qm;
      if (qn > best) { best = qn; arg = k; }          // tf.argmax: first maximal index
    }
    const float nsav = a.tvstream[(size_t)b * a.A + arg] - mt;
    float r = a.reward[b];
    if (a.clip) r = fminf(fmaxf(r, -1.0f), 1.0f);
    const float disc = a.done[b] ? 0.0f : a.discount;
    const float target = nsav * disc + r;
    const float diff = target - sav;
    const float w = a.weight ? a.weight[b] : 1.0f;
    a.target_value[b] = target;
    a.sav[b] = sav;
    const float td = fabsf(diff);
    a.td_dev[b] = td;
    if (a.td_host) a.td_host[b] = td;
    part += diff * diff * w;
    if (a.dq) {
      const float g = -2.0f * w * diff / (float)a.n;
      for (int k = 0; k < a.A; ++k) a.dq[(size_t)b * 32 + k] = (k == act) ? g : 0.f;
      a.dmean[(size_t)b * 32] = -g;
    }
  }
  if (a.loss) {
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += red[i];
      *a.loss = s / (float)a.n;
    }
  }
}

// ------------------------------------------------------------------------------------------
// A3C / A2C losses and head gradients (optimizer/a2c.py:3-26, agent/a3c.py:36-73) on the same network body: the actor
// stream ends in a softmax (model/actor_critic.py:33-34), the critic stream is the scalar value.  Rows [0, n) hold
// network(s, prev_a), rows [n, 2n) network(s', a); next_value is stop_gradient in both losses.
//   adv      = clip(r) + gamma (1 - done) V(s') - V(s)                      (stop_gradient in the policy loss)
//   pi_loss  = -mean(adv * pi(a))        (the probability itself, not its log: optimizer/a2c.py:24)
//   baseline = mean(adv^2) ; entropy = -mean(sum_a -pi log pi)              (no epsilon, like the reference)
//   total    = pi_loss + baseline_coef baseline + entropy_coef entropy
// ------------------------------------------------------------------------------------------
struct A3cArgs {
  const float* policy; const float* value;      // [2n, A], [2n]
  const int32_t* action; const float* reward; const uint8_t* done;
  float discount, baseline_coef, entropy_coef; int clip; int n, A;
  float* adv;                                   // [n] tap
  float* dlogits; float* dv;                    // [n, 32]
  float* loss;                                  // [3] pi, baseline, entropy
};
__global__ void __launch_bounds__(256) a3c_loss_kernel(A3cArgs a) {
  kernel_prologue();
  __shared__ float red[3][8];
  float s_pi = 0.f, s_bl = 0.f, s_en = 0.f;
  const float inv_n = 1.0f / (float)a.n;
  for (int b = threadIdx.x; b < a.n; b += blockDim.x) {
    float r = a.reward[b];
    if (a.clip == DRL_REWARD_ABS_ONE) {
      r = fminf(fmaxf(r, -1.0f), 1.0f);
    } else {                                          // soft_asymmetric (agent/a3c.py:41-43)
      const float sq = tanhf(r / 5.0f);
      r = (r < 0.f ? 0.3f * sq : sq) * 5.0f;
    }
    const float disc = a.done[b] ? 0.0f : a.discount;
    const float adv = r + disc * a.value[a.n + b] - a.value[b];
    a.adv[b] = adv;
    const int act = a.action[b];
    const float* p = a.policy + (size_t)b * a.A;
    float ent = 0.f, sdot = 0.f;
    for (int k = 0; k < a.A; ++k) {
      const float pk = p[k], lp = logf(pk);
      ent += pk * lp;
      const float dpk = ((k == act ? -adv : 0.f) + a.entropy_coef * (lp + 1.0f)) * inv_n;     // d total / d pi_k
      sdot += pk * dpk;
    }
    for (int k = 0; k < a.A; ++k) {                   // through the softmax: dlogit_k = pi_k (dpi_k - sum_j pi_j dpi_j)
      const float pk = p[k];
      const float dpk = ((k == act ? -adv : 0.f) + a.entropy_coef * (logf(pk) + 1.0f)) * inv_n;
      a.dlogits[(size_t)b * 32 + k] = pk * (dpk - sdot);
    }
    a.dv[(size_t)b * 32] = a.baseline_coef * (-2.0f * adv) * inv_n;
    s_pi += (act >= 0 && act < a.A) ? adv * p[act] : 0.f;      // tf.one_hot: an out-of-range action selects nothing
    s_bl += adv * adv;
    s_en += ent;
  }
  s_pi = warp_sum(s_pi); s_bl = warp_sum(s_bl); s_en = warp_sum(s_en);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s_pi; red[1][threadIdx.x >> 5] = s_bl; red[2][threadIdx.x >> 5] = s_en; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t0 = 0.f, t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { t0 += red[0][i]; t1 += red[1][i]; t2 += red[2][i]; }
    a.loss[0] = -t0 * inv_n;
    a.loss[1] = t1 * inv_n;
    a.loss[2] = t2 * inv_n;
  }
}

// ------------------------------------------------------------------------------------------
// Forward of the dueling network (model/apex_value.py:22-41) over M rows.  `tgt` only selects the profile names.
// Weight images (tensor-core modes): img[1]/img[2] conv2/conv3 forward, img[5]/img[6] the dCol operands of backward.
// ------------------------------------------------------------------------------------------

static int apex_forward(const Streams& st, const ApexLayout& pl, const float* P, const WeightImages& wi,
                        const uint8_t* frames, const int32_t* pa, const ApexActs& act, int M, int mode,
                        bool retile_fwd, bool retile_bwd, bool tgt, int* launches) {
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
  // conv1 (model/apex_value.py:5), conv2 (:6), conv3 -> flatten HWC (:7-9), rows in the caller's order
  DRL_TRY(conv_forward_tf32<Geo::IC>(s, pl, P, wi.img[1], wi.img[2], frames, M, 1, act.a1, act.a2, act.a3, mode, tgt,
                                      st.par ? st.ev[7] : nullptr, &n));
  DRL_TRY(join_from_side(st, 1));
  // first layers of both streams: [M, 3392] x [3392, 256 | 256], split-K partial sums, then bias + ReLU (:17-19,28-37)
  const SplitPlan sp = plan_head1(M);
  {
    CatA al{act.a3, act.table, pa};
    DualB bl{P + pl.value1_w, P + pl.mean1_w, Geo::HID, Geo::HID};
    EpRaw<false> ep{act.zpart, kHeadN, (size_t)M * kHeadN, 1.0f, 0, kHeadN};
    GEMM_FFMA(tgt ? "target_heads_l1_fwd" : "heads_l1_fwd", CfgMid, al, bl, ep, M, kHeadN, kCat, sp.splits, sp.kchunk,
              sp.kchunk);
  }
  prof_mark(s, tgt ? "target_heads_l1_bias_relu" : "heads_l1_bias_relu");
  DRL_CUDA_CHECK((launch_k(apex_hid1_kernel, M, 256, 0, s, act.zpart, sp.splits, (size_t)M * kHeadN, P + pl.value1_b,
                           P + pl.mean1_b, act.hid1, M)));
  ++n;
  const size_t head_stride = (size_t)(pl.mean1_w - pl.value1_w);
  {
    PlainA al{act.hid1, Geo::HID, (size_t)M * Geo::HID};
    PlainB bl{P + pl.value2_w, Geo::HID, head_stride};
    EpBiasAct<true, true> ep{act.hid2, Geo::HID, (size_t)M * Geo::HID, P + pl.value2_b, head_stride, 1.0f};
    GEMM_FFMA(tgt ? "target_heads_l2_fwd" : "heads_l2_fwd", CfgSmall, al, bl, ep, M, Geo::HID, Geo::HID, 2, Geo::HID, 0);
  }
  // output layers: value stream [M, A] (final_activation None) and the "mean" stream [M] (:28-39)
  KERNEL(tgt ? "target_heads_out_fwd" : "heads_out_fwd",
         heads_out_forward(s, act.hid2, act.hid2 + (size_t)M * Geo::HID, P + pl.value3_w, P + pl.value3_b,
                           P + pl.mean3_w, P + pl.mean3_b, act.vstream, act.scratch_sm, act.mstream, M, pl.A), 1);
  if (launches) *launches += n;
  return DRL_OK;
}

// Backward through main(s, prev_a): rows [0, Mb) of a forward over M rows.
static int apex_backward(const Streams& st, const ApexLayout& pl, const float* P, const WeightImages& wi, float* G,
                         const uint8_t* frames, const int32_t* pa, const ApexActs& act, const ApexBwd& bw, int M, int Mb,
                         int mode, int* launches) {
  cudaStream_t s = st.main;
  const cudaStream_t side = st.par ? st.side : st.main;
  const RowMap map{M, 1};
  const size_t head_stride = (size_t)(pl.mean1_w - pl.value1_w);
  const int A = pl.A;
  int n = 0;
  KERNEL("heads_out_bwd",
         heads_out_backward(s, bw.dq, bw.dmean, P + pl.value3_w, P + pl.mean3_w, act.hid2,
                            act.hid2 + (size_t)M * Geo::HID, bw.dhid2, bw.dhid2 + (size_t)Mb * Geo::HID, Mb, A), 1);
  DRL_TRY(fork_to_side(st, 0));
  s = side;
  {  // d value3 [256(+1), A]
    PlainAT al{act.hid2, Geo::HID, 0};
    PlainB bl{bw.dq, 32, 0};
    EpRaw<true> ep{G + pl.value3_w, A, 0, 1.0f, Geo::HID, A};
    GEMM_FFMA("value3_wgrad", CfgSmall, al, bl, ep, Geo::HID, 32, Mb, 1, Mb, 0);
  }
  {  // d mean3 [256(+1), 1]
    PlainAT al{act.hid2 + (size_t)M * Geo::HID, Geo::HID, 0};
    PlainB bl{bw.dmean, 32, 0};
    EpRaw<true> ep{G + pl.mean3_w, 1, 0, 1.0f, Geo::HID, 1};
    GEMM_FFMA("mean3_wgrad", CfgSmall, al, bl, ep, Geo::HID, 32, Mb, 1, Mb, 0);
  }
  {  // d {value2, mean2} = hid1^T dhid2
    PlainAT al{act.hid1, Geo::HID, (size_t)M * Geo::HID};
    PlainB bl{bw.dhid2, Geo::HID, (size_t)Mb * Geo::HID};
    EpRaw<true> ep{G + pl.value2_w, Geo::HID, head_stride, 1.0f, Geo::HID, Geo::HID};
    GEMM_FFMA("heads_l2_wgrad", CfgSmall, al, bl, ep, Geo::HID, Geo::HID, Mb, 2, Mb, 0);
  }
  s = st.main;
  {  // dhid1 = dhid2 W2^T * relu'(hid1)
    PlainA al{bw.dhid2, Geo::HID, (size_t)Mb * Geo::HID};
    PlainBT bl{P + pl.value2_w, Geo::HID, head_stride};
    EpReluMask ep{bw.dhid1, act.hid1, Geo::HID, (size_t)Mb * Geo::HID, (size_t)M * Geo::HID};
    GEMM_FFMA("heads_l2_dgrad", CfgSmall, al, bl, ep, Mb, Geo::HID, Geo::HID, 2, Geo::HID, 0);
  }
  DRL_TRY(fork_to_side(st, 2));
  s = side;
  {  // d {value1, mean1} [3392(+1), 256] = concat^T dhid1 ; bias gradient = column sums
    CatAT al{act.a3, act.table, pa};
    PlainB bl{bw.dhid1, Geo::HID, (size_t)Mb * Geo::HID};
    EpRaw<true> ep{G + pl.value1_w, Geo::HID, head_stride, 1.0f, kCat, Geo::HID};
    GEMM_FFMA("heads_l1_wgrad", CfgBig, al, bl, ep, kCat, Geo::HID, Mb, 2, Mb, 0);
  }
  s = st.main;
  {  // d concat = dhid1_value W1v^T + dhid1_mean W1m^T  -> d a3 (ReLU mask) | d emb rows
    DualA al{bw.dhid1, bw.dhid1 + (size_t)Mb * Geo::HID, Geo::HID, Geo::HID};
    DualBT bl{P + pl.value1_w, P + pl.mean1_w, Geo::HID, Geo::HID};
    EpLstmDx ep{bw.da3, act.a3, bw.du};
    GEMM_FFMA("heads_l1_dgrad", CfgMid, al, bl, ep, Mb, kCat, kHeadN, 1, kHeadN, 0);
  }
  DRL_TRY(fork_to_side(st, 4));
  s = side;
  KERNEL("emb_bwd",
         emb_backward(s, bw.du, pa, act.e1, act.table, P + pl.emb2_w, bw.dpre2, bw.dpre1, G + pl.emb1_w,
                      G + pl.emb1_b, G + pl.emb2_w, G + pl.emb2_b, bw.wg_part, Mb, M, 1, A), 4);
  DRL_TRY(conv_backward_tf32<Geo::IC>(st, pl, P, wi, G, frames, map, Mb, act, bw, mode, &n));
  DRL_TRY(join_from_side(st, 6));
  if (launches) *launches += n;
  return DRL_OK;
}

}  // namespace drl

using namespace drl;

namespace {

constexpr const char* kName = "apex";

int alloc_acts(drl_apex* h, ApexActs& a, int cap) {
  const size_t M = cap, A = h->A;
  a.cap = cap;
  DRL_TRY(alloc_trunk_acts(h, a, M, A));
  size_t zmax = 0;
  for (int m = 1; m <= cap; ++m) zmax = std::max(zmax, (size_t)plan_head1(m).splits * m * kHeadN);
  DRL_TRY(dev_alloc(h, &a.zpart, zmax));
  DRL_TRY(dev_alloc(h, &a.hid1, 2 * M * Geo::HID));
  DRL_TRY(dev_alloc(h, &a.hid2, 2 * M * Geo::HID));
  DRL_TRY(dev_alloc(h, &a.vstream, M * A));
  DRL_TRY(dev_alloc(h, &a.scratch_sm, M * A));
  DRL_TRY(dev_alloc(h, &a.mstream, M));
  return DRL_OK;
}

}  // namespace

int drl::enqueue_forward_td(drl_apex* h, const ApexIn& sl, int n, bool train, float* td_host, int* launches) {
  const Streams st = h->streams(), tst = h->target_streams();
  if (h->algo == 1) {      // A3C: one scope; rows [0, n) = network(s, prev_a), rows [n, 2n) = network(s', a)
    DRL_TRY(apex_forward(st, h->pl, h->params, h->wi, sl.frames, sl.pa2, h->act, 2 * n, h->mode, h->images_stale,
                         h->images_stale, false, launches));
    h->images_stale = false;
    A3cArgs a{};
    a.policy = h->act.scratch_sm; a.value = h->act.mstream;
    a.action = sl.pa2 + n; a.reward = sl.reward; a.done = sl.done;
    a.discount = h->cfg.discount_factor; a.baseline_coef = h->a3c_baseline_coef; a.entropy_coef = h->a3c_entropy_coef;
    a.clip = h->a3c_clip; a.n = n; a.A = h->A;
    a.adv = h->adv; a.dlogits = h->bwd.dq; a.dv = h->bwd.dmean; a.loss = h->loss;
    prof_mark(h->compute, "a2c_losses");
    DRL_CUDA_CHECK((launch_k(a3c_loss_kernel, 1, 256, 0, h->compute, a)));
    if (launches) *launches += 1;
    return DRL_OK;
  }
  // the target forward has no dependence on the main forward: fork it onto its own stream pair first, join before the
  // TD kernel (inside a captured step these become parallel branches of the graph)
  if (h->par) {
    DRL_CUDA_CHECK(cudaEventRecord(h->ev_tfork, h->compute));
    DRL_CUDA_CHECK(cudaStreamWaitEvent(h->tmain, h->ev_tfork, 0));
  }
  DRL_TRY(apex_forward(tst, h->pl, h->target, h->twi, sl.frames + (size_t)n * Geo::FRAME, sl.pa2 + n, h->tact, n, h->mode,
                       h->target_images_stale, false, true, launches));
  h->target_images_stale = false;
  if (h->par) DRL_CUDA_CHECK(cudaEventRecord(h->ev_tjoin, h->tmain));
  // rows [0, n) = s with previous_action, rows [n, 2n) = s' with action: one main-network forward covers both
  DRL_TRY(apex_forward(st, h->pl, h->params, h->wi, sl.frames, sl.pa2, h->act, 2 * n, h->mode, h->images_stale,
                       h->images_stale, false, launches));
  h->images_stale = false;
  if (h->par) DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, h->ev_tjoin, 0));
  TdArgs a{};
  a.vstream = h->act.vstream; a.mstream = h->act.mstream;
  a.tvstream = h->tact.vstream; a.tmstream = h->tact.mstream;
  a.action = sl.pa2 + n; a.reward = sl.reward; a.done = sl.done; a.weight = sl.weight;
  a.discount = h->cfg.discount_factor; a.clip = (h->cfg.reward_clipping == DRL_REWARD_ABS_ONE) ? 1 : 0;
  a.n = n; a.A = h->A;
  a.main_q = h->main_q; a.next_main_q = h->next_main_q; a.target_q = h->target_q;
  a.target_value = h->target_value; a.sav = h->sav; a.td_dev = h->td_dev; a.td_host = td_host;
  a.dq = train ? h->bwd.dq : nullptr; a.dmean = train ? h->bwd.dmean : nullptr;
  a.loss = train ? h->loss : nullptr;
  prof_mark(h->compute, "td_target_loss");
  DRL_CUDA_CHECK((launch_k(apex_td_kernel, 1, 256, 0, h->compute, a)));
  if (launches) *launches += 1;
  return DRL_OK;
}

namespace {

int fwd_bwd(LearnerCore* core, int slot, int* launches) {
  drl_apex* h = static_cast<drl_apex*>(core);
  const ApexIn& sl = h->in[slot];
  const int B = h->B;
  DRL_TRY(enqueue_forward_td(h, sl, B, true, h->d_td + (size_t)slot * B, launches));
  return apex_backward(h->streams(), h->pl, h->params, h->wi, h->grads, sl.frames, sl.pa2, h->act, h->bwd, 2 * B, B,
                       h->mode, launches);
}

int stage_into(drl_apex* h, const ApexIn& s, cudaStream_t stream, int n, int row2, const uint8_t* state,
               const uint8_t* next_state, const int32_t* previous_action, const int32_t* action, const float* reward,
               const uint8_t* done, const float* is_weight) {
  auto cp = [&](void* dst, const void* src, size_t bytes) -> cudaError_t {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream);
  };
  DRL_CUDA_CHECK(cp(s.frames, state, (size_t)n * Geo::FRAME));
  if (next_state) DRL_CUDA_CHECK(cp(s.frames + (size_t)row2 * Geo::FRAME, next_state, (size_t)n * Geo::FRAME));
  DRL_CUDA_CHECK(cp(s.pa2, previous_action, (size_t)n * 4));
  if (action) DRL_CUDA_CHECK(cp(s.pa2 + row2, action, (size_t)n * 4));
  if (reward) DRL_CUDA_CHECK(cp(s.reward, reward, (size_t)n * 4));
  if (done) DRL_CUDA_CHECK(cp(s.done, done, (size_t)n));
  // no weights = unit weights (Agent.train, agent/apex.py:167): the slot always holds a weight vector, so a captured
  // graph never depends on which entry point fed it
  if (reward) DRL_CUDA_CHECK(cp(s.weight, is_weight ? is_weight : h->h_ones, (size_t)n * 4));
  return DRL_OK;
}

// the scratch slot, staged synchronously on the compute stream, then one main-network forward over n rows
int forward_main(drl_apex* h, int n, const uint8_t* state, const int32_t* previous_action) {
  const ApexIn& s = h->in[h->num_slots];
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  DRL_TRY(stage_into(h, s, h->compute, n, n, state, nullptr, previous_action, nullptr, nullptr, nullptr, nullptr));
  DRL_TRY(apex_forward(h->streams(), h->pl, h->params, h->wi, s.frames, s.pa2, h->act, n, h->mode, h->images_stale,
                       h->images_stale, false, nullptr));
  h->images_stale = false;
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_apex_create(const drl_apex_config* cfg, drl_apex** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || cfg->channels != Geo::IC) {
    set_error("only the reference input geometry 84x84x4 is supported (got %dx%dx%d)", cfg->height, cfg->width, cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->num_action < 2 || cfg->num_action > 32) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  if (cfg->batch < 1) { set_error("batch must be >= 1"); return DRL_ERR_INVALID; }
  if (cfg->math_mode < 0 || cfg->math_mode > 2) { set_error("math_mode must be 0 (default), 1 (FP32 FFMA) or 2 (wgmma 3xTF32)"); return DRL_ERR_INVALID; }
  if (drl_device_count() <= cfg->device) { set_error("CUDA device %d not available (no CPU fallback)", cfg->device); return DRL_ERR_CUDA; }
  drl_apex* h = new drl_apex();
  h->cfg = *cfg;
  h->device = cfg->device;
  h->num_slots = cfg->num_slots < 1 ? 2 : cfg->num_slots;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->mode = (cfg->math_mode == 0) ? DRL_DEFAULT_MATH_MODE : cfg->math_mode;
  h->B = cfg->batch; h->A = cfg->num_action;
  h->pl.init(h->A);
  h->layout = &h->pl;
  h->fwd_bwd = fwd_bwd;
  AdamState& o = h->opt;
  o.start_lr = cfg->start_learning_rate; o.end_lr = cfg->end_learning_rate; o.learning_frame = cfg->learning_frame;
  o.clip_norm = cfg->gradient_clip_norm;
  int rc = [&]() -> int {
    const size_t B = h->B, A = h->A;
    size_t off = 0;
    const size_t o_fr = off; off = align_up(off + 2 * B * Geo::FRAME, 256);
    const size_t o_pa = off; off = align_up(off + 2 * B * 4, 256);
    const size_t o_rw = off; off = align_up(off + B * 4, 256);
    const size_t o_dn = off; off = align_up(off + B, 256);
    const size_t o_wt = off; off = align_up(off + B * 4, 256);
    DRL_TRY(adam_learner_init(h, off, B));
    for (const LearnerSlot& s : h->slots)
      h->in.push_back(ApexIn{s.base + o_fr, reinterpret_cast<int32_t*>(s.base + o_pa),
                             reinterpret_cast<float*>(s.base + o_rw), s.base + o_dn,
                             reinterpret_cast<float*>(s.base + o_wt)});
    DRL_TRY(alloc_acts(h, h->act, 2 * h->B));
    DRL_TRY(alloc_acts(h, h->tact, h->B));
    ApexBwd& b = h->bwd;
    DRL_TRY(dev_alloc(h, &b.dq, B * 32));
    DRL_TRY(dev_alloc(h, &b.dmean, B * 32));
    DRL_TRY(dev_alloc(h, &b.dhid2, 2 * B * Geo::HID));
    DRL_TRY(dev_alloc(h, &b.dhid1, 2 * B * Geo::HID));
    DRL_TRY(alloc_trunk_bwd(h, b, B, A, Geo::IC, true));
    DRL_TRY(dev_alloc(h, &h->main_q, B * A));
    DRL_TRY(dev_alloc(h, &h->next_main_q, B * A));
    DRL_TRY(dev_alloc(h, &h->target_q, B * A));
    DRL_TRY(dev_alloc(h, &h->target_value, B));
    DRL_TRY(dev_alloc(h, &h->sav, B));
    DRL_TRY(dev_alloc(h, &h->td_dev, B));
    DRL_TRY(dev_alloc(h, &h->adv, B));
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_apex_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_apex_destroy(drl_apex* h) {
  if (!h) return DRL_OK;
  adam_learner_release(h);
  delete h;
  return DRL_OK;
}

int drl_apex_param_count(const drl_apex* h, int64_t* n) { return learner_param_count(h, kName, n); }
int drl_apex_set_params(drl_apex* h, int32_t which, const float* host_flat, int64_t n) {
  return adam_set_params(h, kName, which, host_flat, n);
}
int drl_apex_get_params(drl_apex* h, int32_t which, float* host_flat, int64_t n) {
  return adam_get_params(h, kName, which, host_flat, n);
}
int drl_apex_set_opt_state(drl_apex* h, const float* host_m, const float* host_v, int64_t n, int64_t step,
                           float beta1_power, float beta2_power) {
  return adam_set_opt_state(h, kName, host_m, host_v, n, step, beta1_power, beta2_power);
}
int drl_apex_get_opt_state(drl_apex* h, float* host_m, float* host_v, int64_t n, int64_t* step, float* beta1_power,
                           float* beta2_power) {
  return adam_get_opt_state(h, kName, host_m, host_v, n, step, beta1_power, beta2_power);
}
int drl_apex_get_grads(drl_apex* h, float* host_flat, int64_t n) { return learner_get_grads(h, kName, h->grads, host_flat, n); }
int drl_apex_target_to_main(drl_apex* h) { return adam_main_to_target(h, kName); }   // target <- main (sic)

int drl_apex_stage(drl_apex* h, int32_t slot, const uint8_t* state, const uint8_t* next_state,
                   const int32_t* previous_action, const int32_t* action, const float* reward, const uint8_t* done,
                   const float* is_weight) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  if (!state || !next_state || !previous_action || !action || !reward || !done) { set_error("stage: null input pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  LearnerSlot& s = h->slots[slot];
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, s.consumed, 0));
  DRL_TRY(stage_into(h, h->in[slot], h->copy, h->B, h->B, state, next_state, previous_action, action, reward, done,
                     is_weight));
  DRL_CUDA_CHECK(cudaEventRecord(s.staged, h->copy));
  s.has_data = true;
  return DRL_OK;
}

int drl_apex_step_async(drl_apex* h, int32_t slot) { return learner_step_async(h, kName, slot); }
int drl_apex_forward_backward(drl_apex* h, int32_t slot) { return learner_forward_backward(h, kName, slot); }
int drl_apex_grad_bucket(drl_apex* h, void** dev_ptr, int64_t* count) { return learner_grad_bucket(h, kName, dev_ptr, count); }
int drl_apex_apply(drl_apex* h, float grad_scale) { return learner_apply(h, kName, grad_scale); }

int drl_apex_wait(drl_apex* h, drl_apex_out* out, float* td_error) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);     // the scalar row stays valid while it is read
  const float* r = nullptr;
  DRL_TRY(adam_wait(h, kName, &r, td_error));
  if (out) {
    out->loss = r[0];
    out->learning_rate = r[1];
    out->grad_norm = r[2];
    out->step = step_of(r);
  }
  return DRL_OK;
}

int drl_apex_step(drl_apex* h, int32_t slot, drl_apex_out* out, float* td_error) {
  DRL_TRY(drl_apex_step_async(h, slot));
  return drl_apex_wait(h, out, td_error);
}

int drl_apex_td_error(drl_apex* h, int32_t n, const uint8_t* state, const uint8_t* next_state,
                      const int32_t* previous_action, const int32_t* action, const float* reward, const uint8_t* done,
                      float* td_error) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > h->B) { set_error("td_error: n must be in [1, %d]", h->B); return DRL_ERR_INVALID; }
  if (!state || !next_state || !previous_action || !action || !reward || !done || !td_error) { set_error("td_error: null pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  const ApexIn& s = h->in[h->num_slots];      // scratch slot
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  // rows [0, n) = s, rows [n, 2n) = s' (packed, so that one main-network forward covers both)
  DRL_TRY(stage_into(h, s, h->compute, n, n, state, next_state, previous_action, action, reward, done, nullptr));
  const Streams st = h->streams();
  DRL_TRY(apex_forward(st, h->pl, h->params, h->wi, s.frames, s.pa2, h->act, 2 * n, h->mode, h->images_stale,
                       h->images_stale, false, nullptr));
  h->images_stale = false;
  DRL_TRY(apex_forward(st, h->pl, h->target, h->twi, s.frames + (size_t)n * Geo::FRAME, s.pa2 + n, h->tact, n, h->mode,
                       h->target_images_stale, false, true, nullptr));
  h->target_images_stale = false;
  TdArgs a{};
  a.vstream = h->act.vstream; a.mstream = h->act.mstream;
  a.tvstream = h->tact.vstream; a.tmstream = h->tact.mstream;
  a.action = s.pa2 + n; a.reward = s.reward; a.done = s.done; a.weight = nullptr;
  a.discount = h->cfg.discount_factor; a.clip = (h->cfg.reward_clipping == DRL_REWARD_ABS_ONE) ? 1 : 0;
  a.n = n; a.A = h->A;
  a.main_q = h->main_q; a.next_main_q = h->next_main_q; a.target_q = h->target_q;
  a.target_value = h->target_value; a.sav = h->sav; a.td_dev = h->td_dev; a.td_host = nullptr;
  DRL_CUDA_CHECK((launch_k(apex_td_kernel, 1, 256, 0, h->compute, a)));
  DRL_CUDA_CHECK(cudaMemcpyAsync(td_error, h->td_dev, (size_t)n * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  h->last_n = n;
  return DRL_OK;
}

int drl_apex_act(drl_apex* h, int32_t n, const uint8_t* state, const int32_t* previous_action, float* q_value) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > 2 * h->B) { set_error("act: n must be in [1, %d]", 2 * h->B); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !q_value) { set_error("act: null pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_TRY(forward_main(h, n, state, previous_action));
  const int A = h->A;
  std::vector<float> v((size_t)n * A), m((size_t)n);
  DRL_CUDA_CHECK(cudaMemcpyAsync(v.data(), h->act.vstream, v.size() * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaMemcpyAsync(m.data(), h->act.mstream, m.size() * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < A; ++k) q_value[(size_t)i * A + k] = v[(size_t)i * A + k] - m[i];   // model/apex_value.py:40
  h->last_n = 0;
  return DRL_OK;
}

int drl_apex_taps(drl_apex* h, float* main_q, float* next_main_q, float* target_q, float* target_value,
                  float* state_action_value) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  if (h->last_n < 1) { set_error("taps: no step or td_error call has run"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  const size_t n = h->last_n, A = h->A;
  if (main_q) DRL_CUDA_CHECK(cudaMemcpy(main_q, h->main_q, n * A * 4, cudaMemcpyDeviceToHost));
  if (next_main_q) DRL_CUDA_CHECK(cudaMemcpy(next_main_q, h->next_main_q, n * A * 4, cudaMemcpyDeviceToHost));
  if (target_q) DRL_CUDA_CHECK(cudaMemcpy(target_q, h->target_q, n * A * 4, cudaMemcpyDeviceToHost));
  if (target_value) DRL_CUDA_CHECK(cudaMemcpy(target_value, h->target_value, n * 4, cudaMemcpyDeviceToHost));
  if (state_action_value) DRL_CUDA_CHECK(cudaMemcpy(state_action_value, h->sav, n * 4, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_apex_read_buffer(drl_apex* h, const char* name, float* host_dst, int64_t n) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!name || !host_dst) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  if (h->last_n < 1) { set_error("read_buffer: no step or td_error call has run"); return DRL_ERR_STATE; }
  const size_t Mb = h->last_n, M = 2 * Mb, A = h->A;
  const NamedBuffer tab[] = {
      {"a1", h->act.a1, M * 400 * 32}, {"a2", h->act.a2, M * 81 * 64}, {"a3", h->act.a3, M * Geo::FLAT},
      {"emb", h->act.table, A * Geo::EMB}, {"e1", h->act.e1, A * Geo::EMB},
      {"hid1", h->act.hid1, 2 * M * Geo::HID}, {"hid2", h->act.hid2, 2 * M * Geo::HID},
      {"vstream", h->act.vstream, M * A}, {"mstream", h->act.mstream, M}, {"policy", h->act.scratch_sm, M * A},
      {"dq", h->bwd.dq, Mb * 32}, {"dmean", h->bwd.dmean, Mb * 32},
      {"dhid2", h->bwd.dhid2, 2 * Mb * Geo::HID}, {"dhid1", h->bwd.dhid1, 2 * Mb * Geo::HID},
      {"du", h->bwd.du, Mb * Geo::EMB},
      {"da3", h->bwd.da3, Mb * Geo::FLAT}, {"da2", h->bwd.da2, Mb * 81 * 64}, {"da1", h->bwd.da1, Mb * 400 * 32}};
  return read_named_buffer(h, tab, sizeof(tab) / sizeof(tab[0]), name, host_dst, n);
}

// The launch plan of an Ape-X / A3C step over B transitions in math mode `mode` (forward rows 2B, backward rows B), read
// by the per-kernel tests to assert which edges a case reaches: out[0] = split-K count of heads_l1_fwd, out[1..3] =
// split-K count of the conv1 / conv2 / conv3 weight gradients.
int drl_debug_apex_launch_plan(int32_t B, int32_t mode, int32_t* out) {
  if (!out || B < 1 || mode < 1 || mode > 2) { set_error("apex_launch_plan: need out, B >= 1, mode 1 or 2"); return DRL_ERR_INVALID; }
  out[0] = plan_head1(2 * B).splits;
  out[1] = plan_conv1_wgrad(B, mode).splits;
  out[2] = plan_conv2_wgrad(B, mode).splits;
  out[3] = plan_conv3_wgrad(B, mode).splits;
  return DRL_OK;
}

int drl_apex_profile_step(drl_apex* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels,
                          int32_t* count) {
  return learner_profile_step(h, kName, slot, names, names_len, ms, max_kernels, count);
}
int drl_apex_last_step_ms(drl_apex* h, float* ms) { return learner_last_step_ms(h, kName, ms); }
int drl_apex_stream(drl_apex* h, void** stream) { return learner_stream(h, kName, stream); }
int drl_apex_launches_per_step(const drl_apex* h, int32_t* n) { return learner_launches_per_step(h, kName, n); }

// ---- A3C learner: the same handle type with algo = 1 (include/drl_b200.h) ---------------------------------------
int drl_a3c_create(const drl_a3c_config* cfg, drl_a3c** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->reward_clipping != DRL_REWARD_ABS_ONE && cfg->reward_clipping != DRL_REWARD_SOFT_ASYMMETRIC) {
    set_error("reward_clipping must be DRL_REWARD_ABS_ONE or DRL_REWARD_SOFT_ASYMMETRIC");
    return DRL_ERR_INVALID;
  }
  drl_apex_config c{};
  c.batch = cfg->batch; c.height = cfg->height; c.width = cfg->width; c.channels = cfg->channels;
  c.num_action = cfg->num_action; c.discount_factor = cfg->discount_factor;
  c.start_learning_rate = cfg->start_learning_rate; c.end_learning_rate = cfg->end_learning_rate;
  c.learning_frame = cfg->learning_frame; c.gradient_clip_norm = cfg->gradient_clip_norm;
  c.reward_clipping = cfg->reward_clipping; c.device = cfg->device; c.num_slots = cfg->num_slots;
  c.use_cuda_graph = cfg->use_cuda_graph; c.math_mode = cfg->math_mode;
  drl_apex* h = nullptr;
  DRL_TRY(drl_apex_create(&c, &h));
  h->algo = 1;
  h->a3c_baseline_coef = cfg->baseline_loss_coef;
  h->a3c_entropy_coef = cfg->entropy_coef;
  h->a3c_clip = cfg->reward_clipping;
  *out = h;
  return DRL_OK;
}
int drl_a3c_destroy(drl_a3c* h) { return drl_apex_destroy(h); }
int drl_a3c_param_count(const drl_a3c* h, int64_t* n) { return drl_apex_param_count(h, n); }
int drl_a3c_set_params(drl_a3c* h, const float* host_flat, int64_t n) { return drl_apex_set_params(h, DRL_APEX_MAIN, host_flat, n); }
int drl_a3c_get_params(drl_a3c* h, float* host_flat, int64_t n) { return drl_apex_get_params(h, DRL_APEX_MAIN, host_flat, n); }
int drl_a3c_set_opt_state(drl_a3c* h, const float* m, const float* v, int64_t n, int64_t step, float b1p, float b2p) {
  return drl_apex_set_opt_state(h, m, v, n, step, b1p, b2p);
}
int drl_a3c_get_opt_state(drl_a3c* h, float* m, float* v, int64_t n, int64_t* step, float* b1p, float* b2p) {
  return drl_apex_get_opt_state(h, m, v, n, step, b1p, b2p);
}
int drl_a3c_get_grads(drl_a3c* h, float* host_flat, int64_t n) { return drl_apex_get_grads(h, host_flat, n); }
int drl_a3c_stage(drl_a3c* h, int32_t slot, const uint8_t* state, const uint8_t* next_state, const int32_t* previous_action,
                  const int32_t* action, const float* reward, const uint8_t* done) {
  return drl_apex_stage(h, slot, state, next_state, previous_action, action, reward, done, nullptr);
}
int drl_a3c_stage_from_queue(drl_a3c* h, int32_t slot, drl_a3c_queue* q, int32_t timeout_ms) {
  DRL_TRY(check_handle(h, kName));
  if (!q) { set_error("null a3c queue handle"); return DRL_ERR_INVALID; }
  {
    std::lock_guard<std::recursive_mutex> lk(h->mu);
    if (h->algo != 1) { set_error("stage_from_queue: not an A3C handle"); return DRL_ERR_INVALID; }
    DRL_TRY(check_slot(h, slot));
    if (q->device != h->device) {
      set_error("stage_from_queue: the queue is on device %d, the learner on device %d", q->device, h->device);
      return DRL_ERR_INVALID;
    }
    if (q->T != h->B || q->A != h->A) {
      set_error("stage_from_queue: the queue has trajectory %d, num_action %d; the learner batch %d, num_action %d",
                q->T, q->A, h->B, h->A);
      return DRL_ERR_INVALID;
    }
  }
  // wait for a record without the learner's lock: actor threads sync their engines from this learner meanwhile
  int qs = 0;
  std::vector<cudaEvent_t> ev_commit;
  DRL_TRY(traj_queue_pop(q, timeout_ms, &qs, &ev_commit));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  NvtxRange nv("drl:a3c_stage_from_queue");
  LearnerSlot& s = h->slots[slot];
  const ApexIn& in = h->in[slot];
  const int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(h->device));
    // do not overwrite a slot the compute stream is still reading; do not read a record whose commit copies are pending
    DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, s.consumed, 0));
    for (cudaEvent_t e : ev_commit) DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, e, 0));
    // the queue slot is an ApexIn of B = T rows: field by field, the same bytes drl_a3c_stage uploads
    void* const dst[kApexQFields] = {in.frames, in.pa2, in.reward, in.done};
    for (int f = 0; f < kApexQFields; ++f)
      DRL_CUDA_CHECK(cudaMemcpyAsync(dst[f], q->field(qs, f), q->sz[f], cudaMemcpyDeviceToDevice, h->copy));
    // unit weights, as stage_into stages them: a captured graph never depends on which entry point fed the slot
    DRL_CUDA_CHECK(cudaMemcpyAsync(in.weight, h->h_ones, (size_t)h->B * 4, cudaMemcpyHostToDevice, h->copy));
    DRL_CUDA_CHECK(cudaEventRecord(s.staged, h->copy));
    s.has_data = true;
    return DRL_OK;
  }();
  // the queue slot goes back to the producers either way (their copies into it wait for its release event)
  const int rc_release = traj_queue_release(q, qs, h->copy);
  return rc != DRL_OK ? rc : rc_release;
}
int drl_a3c_step_async(drl_a3c* h, int32_t slot) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->algo != 1) { set_error("not an A3C handle"); return DRL_ERR_INVALID; }
  return drl_apex_step_async(h, slot);
}
int drl_a3c_forward_backward(drl_a3c* h, int32_t slot) { return drl_apex_forward_backward(h, slot); }
int drl_a3c_grad_bucket(drl_a3c* h, void** dev_ptr, int64_t* count) { return drl_apex_grad_bucket(h, dev_ptr, count); }
int drl_a3c_apply(drl_a3c* h, float grad_scale) { return drl_apex_apply(h, grad_scale); }
int drl_a3c_wait(drl_a3c* h, drl_a3c_out* out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);     // the scalar row stays valid while it is read
  const float* r = nullptr;
  DRL_TRY(adam_wait(h, kName, &r, nullptr));
  if (out) {
    out->pi_loss = r[0]; out->baseline_loss = r[3]; out->entropy = r[4];
    out->learning_rate = r[1]; out->grad_norm = r[2]; out->step = step_of(r);
  }
  return DRL_OK;
}
int drl_a3c_step(drl_a3c* h, int32_t slot, drl_a3c_out* out) {
  DRL_TRY(drl_a3c_step_async(h, slot));
  return drl_a3c_wait(h, out);
}
int drl_a3c_act(drl_a3c* h, int32_t n, const uint8_t* state, const int32_t* previous_action, float* policy, float* value) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > 2 * h->B) { set_error("act: n must be in [1, %d]", 2 * h->B); return DRL_ERR_INVALID; }
  if (!state || !previous_action) { set_error("act: null pointer"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_TRY(forward_main(h, n, state, previous_action));
  if (policy) DRL_CUDA_CHECK(cudaMemcpyAsync(policy, h->act.scratch_sm, (size_t)n * h->A * 4, cudaMemcpyDeviceToHost, h->compute));
  if (value) DRL_CUDA_CHECK(cudaMemcpyAsync(value, h->act.mstream, (size_t)n * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  h->last_n = 0;
  return DRL_OK;
}
int drl_a3c_taps(drl_a3c* h, float* policy, float* value, float* next_value, float* advantage) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  if (h->last_n < 1) { set_error("taps: no step has run"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  const size_t n = h->last_n, A = h->A;
  if (policy) DRL_CUDA_CHECK(cudaMemcpy(policy, h->act.scratch_sm, n * A * 4, cudaMemcpyDeviceToHost));
  if (value) DRL_CUDA_CHECK(cudaMemcpy(value, h->act.mstream, n * 4, cudaMemcpyDeviceToHost));
  if (next_value) DRL_CUDA_CHECK(cudaMemcpy(next_value, h->act.mstream + n, n * 4, cudaMemcpyDeviceToHost));
  if (advantage) DRL_CUDA_CHECK(cudaMemcpy(advantage, h->adv, n * 4, cudaMemcpyDeviceToHost));
  return DRL_OK;
}
int drl_a3c_read_buffer(drl_a3c* h, const char* name, float* host_dst, int64_t n) { return drl_apex_read_buffer(h, name, host_dst, n); }
int drl_a3c_profile_step(drl_a3c* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels, int32_t* count) {
  return drl_apex_profile_step(h, slot, names, names_len, ms, max_kernels, count);
}
int drl_a3c_stream(drl_a3c* h, void** stream) { return drl_apex_stream(h, stream); }
int drl_a3c_launches_per_step(const drl_a3c* h, int32_t* n) { return drl_apex_launches_per_step(h, n); }

}  // extern "C"

int drl::apex_params_snapshot(drl_apex* h, int device, int algo, int num_action, cudaStream_t dst_stream, float* dst,
                              cudaEvent_t ev_ready, cudaEvent_t ev_copied) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->algo != algo || h->A != num_action) {
    set_error("sync: the learner is %s with num_action %d, the policy %s with %d", h->algo ? "A3C" : "Ape-X", h->A,
              algo ? "A3C" : "Ape-X", num_action);
    return DRL_ERR_INVALID;
  }
  return learner_params_snapshot(h, kName, device, dst_stream, dst, ev_ready, ev_copied);
}
