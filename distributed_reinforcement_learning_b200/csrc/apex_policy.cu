// apex_policy.cu -- the Ape-X / A3C policy engine behind drl_apex_policy_* and drl_a3c_policy_act (include/drl_b200.h):
// the actor side of train_apex.py:157-231 and train_a3c.py:112-183.  A forward-only handle that runs the shared network
// body (model/apex_value.py:22-40, model/actor_critic.py:27-38) for n <= 64 environments per call and applies the
// action rule of the family's get_policy_and_action on the GPU:
//   algo 0 (Ape-X, agent/apex.py:88-102)  q = value stream - "mean" stream; the first maximum of q, unless the host's
//                                         epsilon draw gave the row an explore action; returns q, action, q[action]
//   algo 1 (A3C, agent/a3c.py:109-119)    policy = softmax(actor stream); numpy's RandomState.choice(A, p=policy) for
//                                         the host's uniform draw; returns policy, action, policy[action].  The critic
//                                         stream is never evaluated (the reference actor fetches only the policy).
//
// One call = one H2D of the staged inputs + 5 kernels on the engine's own stream:
//   conv1 / conv2 / conv3   the Ape-X learner's math-mode-2 kernels and configurations (layer_defs.cuh: conv_forward_tf32)
//   skinny_splitk_fwd       z = [a3 | table[pa]] [W1_value | W1_mean] (Ape-X, N = 512) or [a3 | table[pa]] W1_actor
//                           (A3C, N = 256) as a skinny split-K FP32-FFMA GEMM (K = 3392, policy_lstm.cuh)
//   apex_policy_head        split-K sum + bias + ReLU, the 256 x 256 layer(s), the output layer(s) and the action rule;
//                           writes q / policy, action and q[action] / policy[action] straight into mapped pinned
//                           memory (no D2H node)
// Both new kernels sum in a fixed order without atomics: eager and graph replays, and repeated calls, are bitwise equal.
// The act enqueues two halves: the H2D of its pinned input block, then the kernels on the device input block
// (apex_policy_enqueue_forward), which the A3C policy server (a3c_policy_server.cu) runs on input rows its own kernel
// fills.
//
// The A3C recorder (drl_a3c_policy_recorder_*, DESIGN.md section 15) runs this act unchanged and then one more kernel,
// a3c_record_step, that writes the step into its staging of n unrolls in the device A3C queue's record layout.
#include <string.h>

#include "apex_defs.cuh"
#include "policy_core.cuh"
#include "policy_head.cuh"
#include "policy_lstm.cuh"
#include "queue_recorder.cuh"

namespace drl {
namespace {

constexpr const char* kName = "apex policy";
constexpr int kMaxApexPolicyRows = 64;
constexpr int kApexMaxA = 32;

// ---- skinny_splitk_fwd (policy_lstm.cuh) ------------------------------------------------------------------------
// K = 3392 = 2^6 * 53.  grid (N / 128 column chunks) x (kApexSplits K splits): Ape-X 4 x 53 = 212 CTAs, A3C 2 x 53 =
// 106 CTAs, all resident at once on the 132 SMs of an H100 (<= 48 KB of shared memory each); each CTA streams its
// 64 x 128 fp32 slab of W (32 KB) once, on 4 mbarrier stages of 16 rows.
constexpr int kApexSplits = 53;
constexpr int kApexStages = 4;

template <int kAlgo>
struct ApexAlgo {
  static constexpr int kStreams = kAlgo == 0 ? 2 : 1;   // Ape-X: value and "mean" streams; A3C: the actor stream
  static constexpr int N = kStreams * Geo::HID;         // first-layer columns
};

template <int kAlgo>
int launch_head1(cudaStream_t s, const float* a3, const float* table, const int32_t* pa, const float* w,
                 const float* w2, float* zpart, int n) {
  return launch_skinny_splitk<0, ApexAlgo<kAlgo>::N, kApexSplits, kApexStages, Geo::HID>(s, a3, table, pa, nullptr, w,
                                                                                          w2, zpart, n);
}

// ---- apex_policy_head -------------------------------------------------------------------------------------------
// One CTA per kHR = 8 rows, 256 threads, so the second- and third-layer weights are read from L2 once per 8 rows.
//   layer 1: thread j sums column j of each stream over the splits in index order, adds the bias, applies ReLU;
//   layer 2: dense256_relu per stream (policy_head.cuh, the IMPALA head's layer);
//   layer 3: warp r = row r in the lane layout of heads_out_forward_kernel (lane owns k = lane + 32 i, one chain per
//            action, warp_sum); the Ape-X q = (v + b_v) - mean, the A3C softmax is the learner's (max, expf(l - max),
//            warp_sum, divide);
//   action:  Ape-X the first maximum of q (np.argmax) or the row's explore action; A3C sample_choice (policy_head.cuh).
constexpr int kApexHeadThreads = 256;

template <int kAlgo>
constexpr size_t apex_head_smem() {   // hid1, hid2 [kStreams][kHR][256] | K partials [4][kHR][256] | W3 [256][A] | w_mean3
  return (size_t)(2 * ApexAlgo<kAlgo>::kStreams * kHR * 256 + 4 * kHR * 256 + Geo::HID * kApexMaxA + Geo::HID) * 4;
}

struct ApexHeadArgs {
  const float* zpart;          // [kApexSplits][n][N]
  const float *b1v, *b1m;      // first-layer biases (value / actor, mean)
  const float *w2v, *b2v, *w2m, *b2m;
  const float *w3v, *b3v, *w3m, *b3m;
  const int32_t* explore;      // Ape-X: [n], -1 greedy, otherwise the action
  const double* uniform;       // A3C: [n] in [0, 1)
  float* out;                  // mapped outputs: q or policy [n][A]
  int32_t* action;             // [n]
  float* out_action;           // [n]: q[action] or policy[action]
  int n, A;
};

template <int kAlgo>
__global__ void __launch_bounds__(kApexHeadThreads, 1) apex_policy_head_kernel(const ApexHeadArgs a) {
  constexpr int kStreams = ApexAlgo<kAlgo>::kStreams, N = ApexAlgo<kAlgo>::N;
  kernel_prologue();
  extern __shared__ __align__(16) float hs[];
  float* shid1 = hs;                              // [kStreams][kHR][256]
  float* shid2 = shid1 + kStreams * kHR * 256;    // [kStreams][kHR][256]
  float* part = shid2 + kStreams * kHR * 256;     // [4][kHR][256]
  float* sw3 = part + 4 * kHR * 256;              // value3 / actor3 [256][A], then mean3 [256] (Ape-X)
  const int tid = threadIdx.x, row0 = blockIdx.x * kHR;
  const int nr = min(kHR, a.n - row0), A = a.A;
  // the output layer's weights first: their loads overlap the first two layers
  for (int i = tid; i < Geo::HID * A / 4; i += kApexHeadThreads)
    reinterpret_cast<float4*>(sw3)[i] = ldg4(a.w3v + 4 * i);
  if (kAlgo == 0) sw3[Geo::HID * A + tid] = __ldg(a.w3m + tid);
#pragma unroll
  for (int z = 0; z < kStreams; ++z) {
    const float bias = __ldg((z == 0 ? a.b1v : a.b1m) + tid);
    for (int r = 0; r < kHR; ++r) {
      float v = 0.f;
      if (r < nr) {
        const float* zp = a.zpart + (size_t)(row0 + r) * N + z * Geo::HID + tid;
        float acc = 0.f;
#pragma unroll 8
        for (int s = 0; s < kApexSplits; ++s) acc += zp[(size_t)s * a.n * N];
        v = fmaxf(acc + bias, 0.f);
      }
      shid1[(z * kHR + r) * 256 + tid] = v;
    }
  }
  __syncthreads();
  dense256_relu(shid1, a.w2v, a.b2v, part, shid2, tid);
  if (kAlgo == 0) dense256_relu(shid1 + kHR * 256, a.w2m, a.b2m, part, shid2 + kHR * 256, tid);
  const int warp = tid >> 5, lane = tid & 31;
  if (warp >= nr) return;
  const int m = row0 + warp;
  float acc[kApexMaxA];
#pragma unroll
  for (int k = 0; k < kApexMaxA; ++k) acc[k] = 0.f;
  float vacc = 0.f;
#pragma unroll
  for (int i = 0; i < Geo::HID / 32; ++i) {
    const int k = lane + 32 * i;
    const float x = shid2[warp * 256 + k];
    if (kAlgo == 0) vacc = fmaf(shid2[(kHR + warp) * 256 + k], sw3[Geo::HID * A + k], vacc);
#pragma unroll
    for (int c = 0; c < kApexMaxA; ++c)
      if (c < A) acc[c] = fmaf(x, sw3[k * A + c], acc[c]);
  }
  float mine = -INFINITY;   // lane c keeps output c
  float mx = -INFINITY;
#pragma unroll
  for (int c = 0; c < kApexMaxA; ++c) {
    if (c < A) {
      const float l = warp_sum(acc[c]) + __ldg(a.b3v + c);
      mx = fmaxf(mx, l);
      if (lane == c) mine = l;
    }
  }
  float* sp = part + warp * 32;      // the K partials are dead after the second dense layer
  if (kAlgo == 0) {
    const float mean = warp_sum(vacc) + __ldg(a.b3m);
    const float q = mine - mean;
    if (lane < A) {
      sp[lane] = q;
      a.out[(size_t)m * A + lane] = q;
    }
    __syncwarp();
    if (lane == 0) {
      float best = sp[0];            // np.argmax: the first maximum
      int arg = 0;
      for (int k = 1; k < A; ++k) {
        if (sp[k] > best) { best = sp[k]; arg = k; }
      }
      const int e = a.explore[m];
      const int act = e >= 0 ? e : arg;
      a.action[m] = act;
      a.out_action[m] = sp[act];
    }
  } else {
    const float e = (lane < A) ? expf(mine - mx) : 0.f;
    const float sum = warp_sum(e);
    const float p = e / sum;
    if (lane < A) a.out[(size_t)m * A + lane] = p;
    sp[lane] = p;
    __syncwarp();
    if (lane == 0) {
      const int act = sample_choice(sp, A, a.uniform, m);
      a.action[m] = act;
      a.out_action[m] = sp[act];
    }
  }
}

// ---- a3c_record_step --------------------------------------------------------------------------------------------
// Step t of the A3C recorder's n unrolls, one CTA per row, 16-byte copies, after the act's head in stream order.  Row i
// of the staging (the queue's record layout, ApexQueueField) gets: state row t <- the act's frame; pa2[t] <- its
// previous action; pa2[T + t] <- the action the head sampled (read from the engine's mapped outputs); and for t >= 1
// next_state row t-1 <- the same frame, or the host's reset frame when the host flagged the row (its previous
// next_state differed from this state: an episode reset).  The step and the flags are read from mapped host memory at
// run time, so one captured graph replays every step; a flagged row's frame crosses PCIe only then.
constexpr int kA3CRecThreads = 256;

struct A3CRecordArgs {
  const uint8_t* frames;       // the act's input frames [n] (engine input block)
  const int32_t* pa;           // [n]
  const int32_t* action;       // [n] the head's actions (mapped)
  const int32_t* ctl;          // mapped: [0] the step t, [1 + i] nonzero when row i's next_state of step t-1 is reset[i]
  const uint8_t* reset;        // mapped [n] frames
  uint8_t* rec_frames;         // staging [n][2T] frames
  int32_t* rec_pa2;            // staging [n][2T]
  int T;
};

__global__ void __launch_bounds__(kA3CRecThreads) a3c_record_step_kernel(const A3CRecordArgs a) {
  kernel_prologue();
  constexpr int kF16 = Geo::FRAME / 16;
  const int row = blockIdx.x, tid = threadIdx.x, t = a.ctl[0];
  const bool from_reset = t > 0 && a.ctl[1 + row] != 0;
  const uint4* f = reinterpret_cast<const uint4*>(a.frames) + (size_t)row * kF16;
  const uint4* fr = reinterpret_cast<const uint4*>(a.reset) + (size_t)row * kF16;
  uint4* st = reinterpret_cast<uint4*>(a.rec_frames) + ((size_t)row * 2 * a.T + t) * kF16;
  uint4* nx = reinterpret_cast<uint4*>(a.rec_frames) + ((size_t)row * 2 * a.T + a.T + t - 1) * kF16;
  const bool next_is_frame = t > 0 && !from_reset;
  for (int i = tid; i < kF16; i += kA3CRecThreads) {
    const uint4 v = f[i];
    st[i] = v;
    if (next_is_frame) nx[i] = v;
  }
  if (from_reset)
    for (int i = tid; i < kF16; i += kA3CRecThreads) nx[i] = fr[i];
  if (tid == 0) {
    a.rec_pa2[(size_t)row * 2 * a.T + t] = a.pa[row];
    a.rec_pa2[(size_t)row * 2 * a.T + a.T + t] = a.action[row];
  }
}

// ---- handle -----------------------------------------------------------------------------------------------------
// device input block of one call with n rows, one contiguous H2D: [frames | previous_action | explore (i32) or uniform
// (f64)]
struct ApexInLayout {
  size_t frames, pa, sel, total;
};
ApexInLayout apex_in_layout(int n) {
  ApexInLayout l;
  size_t off = 0;
  l.frames = off; off = align_up(off + (size_t)n * Geo::FRAME, 256);
  l.pa = off;     off = align_up(off + (size_t)n * 4, 256);
  l.sel = off;    off = align_up(off + (size_t)n * 8, 256);
  l.total = off;
  return l;
}

int set_apex_policy_kernel_attributes() {
  DRL_TRY((set_skinny_splitk_attributes<0, ApexAlgo<0>::N, kApexSplits, kApexStages, Geo::HID>()));
  DRL_TRY((set_skinny_splitk_attributes<0, ApexAlgo<1>::N, kApexSplits, kApexStages, Geo::HID>()));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(apex_policy_head_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)apex_head_smem<0>()));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(apex_policy_head_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)apex_head_smem<1>()));
  return DRL_OK;
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_apex_policy : PolicyCore {
  ApexLayout pl{};
  int algo = 0;   // 0 = Ape-X, 1 = A3C
  // mapped outputs: q / policy [max_batch][A] | action | q[action] / policy[action]
  size_t off_act = 0, off_sel = 0;
};

// the recorder's staging (RecorderCore) is in the A3C queue's field order (ApexQueueField)
struct drl_a3c_policy_recorder : RecorderCore {
  drl_apex_policy* policy = nullptr;
  // mapped pinned block: control words [1 + n] i32 (a3c_record_step_kernel's ctl) | n frames, the reset frames of an
  // act and the final next_state frames of a commit
  uint8_t* h_blk = nullptr;
  uint8_t* d_blk = nullptr;
  size_t off_frames = 0;
  int32_t* ctl() { return reinterpret_cast<int32_t*>(h_blk); }
  uint8_t* frames() { return h_blk + off_frames; }
};

namespace {

// the kernels of the engine's act of n rows on the device input block d_in, writing `out`
int enqueue_forward(drl_apex_policy* h, int n, const ApexPolicyOutRows& out) {
  const ApexInLayout l = apex_in_layout(n);
  const ApexLayout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  DRL_TRY(policy_conv_forward_tf32(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, h->a1, h->a2, h->a3));
  ApexHeadArgs a;
  a.zpart = h->zpart;
  a.b1v = P + pl.value1_b; a.b1m = P + pl.mean1_b;
  a.w2v = P + pl.value2_w; a.b2v = P + pl.value2_b;
  a.w2m = P + pl.mean2_w; a.b2m = P + pl.mean2_b;
  a.w3v = P + pl.value3_w; a.b3v = P + pl.value3_b;
  a.w3m = P + pl.mean3_w; a.b3m = P + pl.mean3_b;
  a.explore = reinterpret_cast<const int32_t*>(h->d_in + l.sel);
  a.uniform = reinterpret_cast<const double*>(h->d_in + l.sel);
  a.out = out.out;
  a.action = out.action;
  a.out_action = out.out_action;
  a.n = n;
  a.A = h->A;
  const int grid = cdiv(n, kHR);
  if (h->algo == 0) {
    DRL_TRY(launch_head1<0>(s, h->a3, h->table, pa, P + pl.value1_w, P + pl.mean1_w, h->zpart, n));
    DRL_CUDA_CHECK((launch_k(apex_policy_head_kernel<0>, grid, kApexHeadThreads, apex_head_smem<0>(), s, a)));
  } else {
    DRL_TRY(launch_head1<1>(s, h->a3, h->table, pa, P + pl.value1_w, nullptr, h->zpart, n));
    DRL_CUDA_CHECK((launch_k(apex_policy_head_kernel<1>, grid, kApexHeadThreads, apex_head_smem<1>(), s, a)));
  }
  return DRL_OK;
}

// the engine's act of n rows: the upload of the staged input block, then its kernels into the mapped outputs
int enqueue_act(PolicyCore* c, int n) {
  drl_apex_policy* h = static_cast<drl_apex_policy*>(c);
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, apex_in_layout(n).total, cudaMemcpyHostToDevice, h->stream));
  const ApexPolicyOutRows out{reinterpret_cast<float*>(h->d_out), reinterpret_cast<int32_t*>(h->d_out + h->off_act),
                              reinterpret_cast<float*>(h->d_out + h->off_sel)};
  return enqueue_forward(h, n, out);
}

// checks common to both act entry points; on success the caller stages `sel` and calls run_act
int check_act(drl_apex_policy* h, int algo, int32_t n, const uint8_t* state, const int32_t* previous_action) {
  if (h->algo != algo) {
    set_error("act: this policy is %s, use %s", h->algo ? "A3C" : "Ape-X",
              h->algo ? "drl_a3c_policy_act" : "drl_apex_policy_act");
    return DRL_ERR_INVALID;
  }
  DRL_TRY(policy_check_n(h, n, state && previous_action));
  return policy_check_actions(h, n, previous_action, nullptr);
}

// stages frames and previous actions (the row selectors are already staged)
void stage_rows(drl_apex_policy* h, int n, const uint8_t* state, const int32_t* previous_action) {
  const ApexInLayout l = apex_in_layout(n);
  memcpy(h->h_in + l.frames, state, (size_t)n * Geo::FRAME);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
}

void copy_outputs(const drl_apex_policy* h, int n, int32_t* action, float* out, float* out_action) {
  if (out) memcpy(out, h->h_out, (size_t)n * h->A * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
  if (out_action) memcpy(out_action, h->h_out + h->off_sel, (size_t)n * 4);
}

// stages frames and previous actions (the row selectors are already staged), runs the call, copies the outputs out
int run_act(drl_apex_policy* h, int n, const uint8_t* state, const int32_t* previous_action, int32_t* action,
            float* out, float* out_action) {
  stage_rows(h, n, state, previous_action);
  DRL_TRY(policy_run_act(h, n));
  copy_outputs(h, n, action, out, out_action);
  return DRL_OK;
}

// drl_a3c_policy_act's checks of its inputs and the staging of its uniforms (the caller holds the engine's lock)
int check_stage_a3c(drl_apex_policy* h, int n, const uint8_t* state, const int32_t* previous_action,
                    const double* uniform) {
  DRL_TRY(check_act(h, 1, n, state, previous_action));
  if (!uniform) { set_error("act: null input pointer (uniform: one draw in [0, 1) per row)"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i) {
    if (!(uniform[i] >= 0.0 && uniform[i] < 1.0)) {
      set_error("act: uniform[%d] = %g is outside [0, 1)", i, uniform[i]);
      return DRL_ERR_INVALID;
    }
  }
  memcpy(h->h_in + apex_in_layout(n).sel, uniform, (size_t)n * 8);
  return DRL_OK;
}

// the recorder's step: the plain act of its n rows, then a3c_record_step
int enqueue_a3c_record(drl_a3c_policy_recorder* r) {
  drl_apex_policy* h = r->policy;
  DRL_TRY(enqueue_act(h, r->n));
  const ApexInLayout l = apex_in_layout(r->n);
  A3CRecordArgs a;
  a.frames = h->d_in + l.frames;
  a.pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  a.action = reinterpret_cast<const int32_t*>(h->d_out + h->off_act);
  a.ctl = reinterpret_cast<const int32_t*>(r->d_blk);
  a.reset = r->d_blk + r->off_frames;
  a.rec_frames = r->field(kApexQFrames);
  a.rec_pa2 = reinterpret_cast<int32_t*>(r->field(kApexQPa2));
  a.T = r->T;
  DRL_CUDA_CHECK((launch_k(a3c_record_step_kernel, r->n, kA3CRecThreads, 0, h->stream, a)));
  return DRL_OK;
}

}  // namespace

namespace drl {

PolicyCore* apex_policy_core_of(drl_apex_policy* h) { return h; }
int apex_policy_algo(const drl_apex_policy* h) { return h->algo; }

ApexPolicyInRows apex_policy_input_rows(drl_apex_policy* h, int n) {
  const ApexInLayout l = apex_in_layout(n);
  return ApexPolicyInRows{h->d_in + l.frames, reinterpret_cast<int32_t*>(h->d_in + l.pa),
                          reinterpret_cast<double*>(h->d_in + l.sel)};
}

int apex_policy_enqueue_forward(drl_apex_policy* h, int n, const ApexPolicyOutRows& out) {
  return enqueue_forward(h, n, out);
}

}  // namespace drl

extern "C" {

int drl_apex_policy_create(const drl_apex_policy_config* cfg, drl_apex_policy** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->max_batch < 1 || cfg->max_batch > kMaxApexPolicyRows) {
    set_error("max_batch must be in [1, %d] (got %d)", kMaxApexPolicyRows, cfg->max_batch);
    return DRL_ERR_INVALID;
  }
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || cfg->channels != Geo::IC) {
    set_error("only the reference input geometry 84x84x4 is supported (got %dx%dx%d)", cfg->height, cfg->width,
              cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->num_action < 2 || cfg->num_action > kApexMaxA) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  if (cfg->algo != 0 && cfg->algo != 1) { set_error("algo must be 0 (Ape-X) or 1 (A3C) (got %d)", cfg->algo); return DRL_ERR_INVALID; }
  DRL_TRY(policy_check_device(cfg->device));
  NvtxRange nv("drl:apex_policy_create");
  drl_apex_policy* h = new drl_apex_policy();
  h->device = cfg->device;
  h->max_batch = cfg->max_batch;
  h->A = cfg->num_action;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->algo = cfg->algo;
  h->pl.init(h->A);
  h->layout = &h->pl;
  h->enqueue_act = enqueue_act;
  h->conv_images = policy_conv_images_tf32;
  const size_t MB = cfg->max_batch;
  h->off_act = align_up(MB * kApexMaxA * 4, 256);
  h->off_sel = h->off_act + align_up(MB * 4, 256);
  const size_t out_bytes = h->off_sel + align_up(MB * 4, 256);
  const size_t N = cfg->algo == 0 ? ApexAlgo<0>::N : ApexAlgo<1>::N;
  h->splits = kApexSplits;
  h->zpart_cols = (int)N;
  const int rc = policy_core_init(h, set_apex_policy_kernel_attributes, kApexSplits * MB * N, apex_in_layout(MB).total,
                                  out_bytes);
  if (rc != DRL_OK) { delete h; return rc; }
  *out = h;
  return DRL_OK;
}

int drl_apex_policy_destroy(drl_apex_policy* h) { return policy_destroy(h); }
int drl_apex_policy_param_count(const drl_apex_policy* h, int64_t* n) { return policy_param_count(h, kName, n); }
int drl_apex_policy_set_params(drl_apex_policy* h, const float* host_flat, int64_t n) {
  return policy_set_params(h, kName, host_flat, n);
}
int drl_apex_policy_get_params(drl_apex_policy* h, float* host_flat, int64_t n) {
  return policy_get_params(h, kName, host_flat, n);
}
int drl_apex_policy_sync_from_learner(drl_apex_policy* h, drl_apex* learner) {
  return policy_sync(h, kName, learner, [&] {
    return apex_params_snapshot(learner, h->device, h->algo, h->A, h->stream, h->params, h->ev_ready, h->ev_copied);
  });
}
int drl_apex_policy_last_act_ms(drl_apex_policy* h, float* ms) { return policy_last_act_ms(h, kName, ms); }
int drl_apex_policy_read_buffer(drl_apex_policy* h, const char* name, float* host_dst, int64_t n) {
  return policy_read_buffer(h, kName, name, host_dst, n);
}
int drl_apex_policy_buffer_dims(drl_apex_policy* h, int32_t* out) { return policy_buffer_dims(h, kName, out); }

int drl_apex_policy_act(drl_apex_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const int32_t* explore_action, int32_t* action, float* q, float* q_action) {
  DRL_TRY(policy_check(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_act(h, 0, n, state, previous_action));
  DRL_TRY(policy_check_actions(h, n, nullptr, explore_action));
  NvtxRange nv("drl:apex_policy_act");
  // the previous call has completed (this entry point is synchronous): the staging block is free
  policy_stage_explore(h->h_in + apex_in_layout(n).sel, explore_action, n);
  return run_act(h, n, state, previous_action, action, q, q_action);
}

int drl_a3c_policy_act(drl_a3c_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                       const double* uniform, int32_t* action, float* policy, float* prob_action) {
  DRL_TRY(policy_check(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_stage_a3c(h, n, state, previous_action, uniform));
  NvtxRange nv("drl:a3c_policy_act");
  return run_act(h, n, state, previous_action, action, policy, prob_action);
}

// ---- A3C recorder -----------------------------------------------------------------------------------------------
int drl_a3c_policy_recorder_destroy(drl_a3c_policy_recorder* r) {
  if (!r) return DRL_OK;
  {
    std::lock_guard<std::recursive_mutex> lk(r->engine->mu);
    cudaSetDevice(r->engine->device);
    recorder_core_release(r);   // waits for the engine's stream: nothing reads h_blk any more
    if (r->h_blk) cudaFreeHost(r->h_blk);
  }
  delete r;
  return DRL_OK;
}

int drl_a3c_policy_recorder_create(drl_a3c_policy* h, drl_a3c_queue* q, int32_t n, drl_a3c_policy_recorder** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  DRL_TRY(policy_check(h, kName));
  if (!q) { set_error("null a3c queue handle"); return DRL_ERR_INVALID; }
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->algo != 1) { set_error("recorder: this policy is Ape-X; an A3C recorder needs an A3C engine (algo 1)"); return DRL_ERR_INVALID; }
  if (n < 1 || n > h->max_batch) {
    set_error("recorder: n must be in [1, %d] (the engine's max_batch; got %d)", h->max_batch, n);
    return DRL_ERR_INVALID;
  }
  if (q->device != h->device) {
    set_error("recorder: the queue is on device %d, the policy on device %d", q->device, h->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != h->A) { set_error("recorder: the queue has num_action %d, the policy %d", q->A, h->A); return DRL_ERR_INVALID; }
  if (n > traj_queue_max_rows(q)) {
    set_error("recorder: %d rows per commit can never fit in the queue (at most %d)", n, traj_queue_max_rows(q));
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:a3c_policy_recorder_create");
  drl_a3c_policy_recorder* r = new drl_a3c_policy_recorder();
  r->engine = r->policy = h;
  r->q = q;
  r->n = n;
  r->T = q->T;
  r->f_reward = kApexQReward;
  r->f_done = kApexQDone;
  r->commit_range = "drl:a3c_policy_recorder_commit";
  const int rc = [&]() -> int {
    DRL_TRY(recorder_core_init(r));
    r->off_frames = align_up((size_t)(1 + n) * 4, 256);
    const size_t bytes = r->off_frames + (size_t)n * Geo::FRAME;
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&r->h_blk, bytes, cudaHostAllocMapped));
    memset(r->h_blk, 0, bytes);
    DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&r->d_blk, r->h_blk, 0));
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    drl_a3c_policy_recorder_destroy(r);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = r;
  return DRL_OK;
}

int drl_a3c_policy_recorder_act(drl_a3c_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                                const double* uniform, const uint8_t* previous_next_state, int32_t* action,
                                float* policy, float* prob_action) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  drl_apex_policy* h = r->policy;
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(recorder_check_step(r));
  DRL_TRY(check_stage_a3c(h, r->n, state, previous_action, uniform));
  if (r->t > 0 && !previous_next_state) {
    set_error("recorder act: null previous_next_state (step %d needs the next_state of step %d)", r->t, r->t - 1);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:a3c_policy_recorder_act");
  // the previous act waited for the stream: the mapped block is free.  A row's next_state of step t-1 is this act's
  // frame unless the environment was reset in between; only then does the host frame go up.
  int32_t* ctl = r->ctl();
  ctl[0] = r->t;
  for (int i = 0; r->t > 0 && i < r->n; ++i) {
    const uint8_t* prev = previous_next_state + (size_t)i * Geo::FRAME;
    ctl[1 + i] = memcmp(prev, state + (size_t)i * Geo::FRAME, Geo::FRAME) != 0;
    if (ctl[1 + i]) memcpy(r->frames() + (size_t)i * Geo::FRAME, prev, Geo::FRAME);
  }
  stage_rows(h, r->n, state, previous_action);
  DRL_TRY(recorder_run_act(r, [r] { return enqueue_a3c_record(r); }));
  copy_outputs(h, r->n, action, policy, prob_action);
  return DRL_OK;
}

int drl_a3c_policy_recorder_commit(drl_a3c_policy_recorder* r, const float* reward, const uint8_t* done,
                                   const uint8_t* next_state, int32_t timeout_ms) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  if (!next_state) { set_error("recorder commit: null argument"); return DRL_ERR_INVALID; }
  // next_state row T-1 of each unroll: the frames env.step returned at step T-1, which no later act sees.  One strided
  // H2D writes row i's frame at its record's last next_state row.
  return recorder_commit(r, reward, done, timeout_ms, [r, next_state]() -> int {
    const size_t F = Geo::FRAME, T = r->T;
    memcpy(r->frames(), next_state, (size_t)r->n * F);   // every act since the last commit waited for the stream
    DRL_CUDA_CHECK(cudaMemcpy2DAsync(r->field(kApexQFrames) + (2 * T - 1) * F, 2 * T * F, r->frames(), F, F, r->n,
                                     cudaMemcpyHostToDevice, r->policy->stream));
    return DRL_OK;
  });
}

int drl_a3c_policy_recorder_reset(drl_a3c_policy_recorder* r) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  return recorder_reset(r);
}

}  // extern "C"
