// policy.cu -- the IMPALA policy engine behind drl_policy_* (include/drl_b200.h): the actor side of train_impala.py:132-194.
// A forward-only handle that runs network() (model/impala_actor_critic.py:33-42, actor head only) for n <= 64
// environments per call and samples each row's action on the GPU (agent/impala.py:118-130).
//
// One call = one H2D of the staged inputs + 5 kernels on the engine's own stream:
//   conv1 / conv2 / conv3   the learner's math-mode-5 kernels and configurations (layers.cu: conv_forward16)
//   policy_lstm_fwd         z = [a3 | table[pa] | h0] W_lstm as a skinny split-K FP32-FFMA GEMM (K = 3648, N = 1024): the
//                           learner's LSTM GEMM is shaped for hundreds of rows (128-row wgmma tiles on a 16-bit weight
//                           image); at n <= 64 the cost is streaming the 14.9 MB of fp32 weights once, over every SM
//   policy_head_fused       split-K sum + bias + gates (c1, h1), actor dense 256 / 256 / A, softmax, sampling; writes
//                           policy, h1, c1 and action straight into mapped pinned memory (no D2H node)
// Both new kernels sum in a fixed order without atomics: eager and graph replays, and repeated calls, are bitwise equal.
//
// A recorder (drl_policy_recorder_*, DESIGN.md section 12) binds the engine to a device trajectory queue
// (traj_queue.cuh).  Its act is the engine's act with policy_head_record in place of policy_head_fused (the same head
// that also writes policy and action into the recorder's staging) plus policy_record_step (frames, previous action,
// h0, c0 of the device input block into the staging); the step t reaches both through a device word staged per call,
// so one graph per recorder replays every step.
#include <string.h>

#include "policy_core.cuh"
#include "policy_head.cuh"
#include "policy_lstm.cuh"
#include "queue_recorder.cuh"

namespace drl {
namespace {

constexpr const char* kName = "policy";
constexpr int kMaxPolicyRows = 64;

// ---- policy_lstm_fwd (policy_lstm.cuh) --------------------------------------------------------------------------
// grid (1024 / kLN column chunks) x (kLSplits K splits) = 8 x 16 = 128 CTAs: one wave on the 132 SMs of an H100, each
// streaming its 228 x 128 fp32 slab of W (114 KB) once.
constexpr int kLSplits = 16;

// ---- policy_head_fused ------------------------------------------------------------------------------------------
// One CTA per kHR rows, 256 threads.  With 8 rows per CTA the 0.54 MB of actor-head weights is read from L2 once per 8
// rows (8 CTAs at n = 64).  The two 256 x 256 layers: thread (q, g) owns columns 4q..4q+3 over the K quarter g, with
// 16 float4 weight loads in flight; the four K partials are added in fixed order (0 + 1) + 2 + 3.  The output layer and
// the softmax: warp r = row r, lane a = logit a (K in four interleaved chains added in fixed order); the softmax is that
// of heads_out_forward_kernel (max, expf(l - max), warp_sum, divide).
constexpr int kHThreads = 256;
constexpr int kMaxA = 32;
// shared memory (floats): h1 / hid2 [kHR][256], hid1 [kHR][256], K partials [4][kHR][256], W3 [256][A <= 32]
constexpr size_t kHeadSmemFloats = 2 * kHR * 256 + 4 * kHR * 256 + 256 * kMaxA;
constexpr size_t kHeadSmem = kHeadSmemFloats * 4;

struct HeadArgs {
  const float* zpart;      // [kLSplits][n][1024]
  const float* lstm_b;     // [1024]
  const float* c0;         // [n][256]
  const double* uniform;   // [n]
  const float *w1, *b1, *w2, *b2, *w3, *b3;   // actor head (fully_connected "actor", :27-30,40)
  float* policy;           // mapped outputs: [n][A]
  float* h1;               // [n][256]
  float* c1;               // [n][256]
  int32_t* action;         // [n]
  int n, A;
};

// what the recording head writes besides HeadArgs' outputs: policy and action of step *t of rows 0..n-1
struct HeadRecord {
  const int32_t* t;        // device word, staged per call
  float* mu;               // [n][T][A]
  int32_t* action;         // [n][T]
  int T;
};

__global__ void __launch_bounds__(kHThreads, 1) policy_head_fused_kernel(const HeadArgs a) {
  kernel_prologue();
  extern __shared__ __align__(16) float hs[];
  float* sh = hs;                    // h1, later hid2
  float* shid = sh + kHR * 256;      // hid1
  float* part = shid + kHR * 256;
  float* sw3 = part + 4 * kHR * 256;
  const int tid = threadIdx.x, row0 = blockIdx.x * kHR;
  const int nr = min(kHR, a.n - row0), A = a.A;
  // the output layer's weights first: their loads overlap the gate math
  for (int i = tid; i < Geo::HID * A / 4; i += kHThreads)
    reinterpret_cast<float4*>(sw3)[i] = ldg4(a.w3 + 4 * i);
  // LSTM cell (TF1 LSTMCell, gate order i, j, f, o, forget bias 1.0): the split partials in fixed order + bias
  {
    const int u = tid;
    float bz[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) bz[g] = __ldg(a.lstm_b + g * Geo::L + u);
    for (int r = 0; r < kHR; ++r) {
      float hv = 0.f;
      if (r < nr) {
        const int m = row0 + r;
        float z[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float acc = 0.f;
#pragma unroll
          for (int s = 0; s < kLSplits; ++s) acc += a.zpart[((size_t)s * a.n + m) * Geo::G4 + g * Geo::L + u];
          z[g] = acc + bz[g];
        }
        const float si = sigmoidf_acc(z[0]);
        const float tj = tanhf(z[1]);
        const float sf = sigmoidf_acc(z[2] + 1.0f);
        const float so = sigmoidf_acc(z[3]);
        const float cv = sf * a.c0[(size_t)m * Geo::L + u] + si * tj;
        hv = so * tanhf(cv);
        a.c1[(size_t)m * Geo::L + u] = cv;
        a.h1[(size_t)m * Geo::L + u] = hv;
      }
      sh[r * 256 + u] = hv;
    }
  }
  __syncthreads();
  dense256_relu(sh, a.w1, a.b1, part, shid, tid);    // hid1
  dense256_relu(shid, a.w2, a.b2, part, sh, tid);    // hid2 (over h1, no longer needed)
  const int warp = tid >> 5, lane = tid & 31;
  if (warp >= nr) return;
  const int m = row0 + warp;
  const float* x = sh + warp * 256;
  float logit = -INFINITY;
  if (lane < A) {
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll 4
    for (int k = 0; k < Geo::HID; k += 4) {
      c0 = fmaf(x[k], sw3[k * A + lane], c0);
      c1 = fmaf(x[k + 1], sw3[(k + 1) * A + lane], c1);
      c2 = fmaf(x[k + 2], sw3[(k + 2) * A + lane], c2);
      c3 = fmaf(x[k + 3], sw3[(k + 3) * A + lane], c3);
    }
    logit = ((c0 + c1) + (c2 + c3)) + __ldg(a.b3 + lane);
  }
  const float mx = warp_max(logit);
  const float e = (lane < A) ? expf(logit - mx) : 0.f;
  const float sum = warp_sum(e);
  const float p = e / sum;
  if (lane < A) a.policy[(size_t)m * A + lane] = p;
  // sampling: numpy's RandomState.choice(A, p=policy) for the row's uniform draw (policy_head.cuh)
  float* sp = part + warp * 32;      // the K partials are dead after the second dense layer
  sp[lane] = p;
  __syncwarp();
  if (lane == 0) a.action[m] = sample_choice(sp, A, a.uniform, m);
}

// The recording head: policy_head_fused_kernel, plus each row's policy and sampled action written into a recorder's
// staging at step *rec.t.  A separate copy rather than a template flag or a shared device function: both of those
// changed the code nvcc generates for policy_head_fused_kernel itself, which the plain act path keeps as it was.
__global__ void __launch_bounds__(kHThreads, 1) policy_head_record_kernel(const HeadArgs a, const HeadRecord rec) {
  kernel_prologue();
  extern __shared__ __align__(16) float hs[];
  float* sh = hs;                    // h1, later hid2
  float* shid = sh + kHR * 256;      // hid1
  float* part = shid + kHR * 256;
  float* sw3 = part + 4 * kHR * 256;
  const int tid = threadIdx.x, row0 = blockIdx.x * kHR;
  const int nr = min(kHR, a.n - row0), A = a.A;
  // the output layer's weights first: their loads overlap the gate math
  for (int i = tid; i < Geo::HID * A / 4; i += kHThreads)
    reinterpret_cast<float4*>(sw3)[i] = ldg4(a.w3 + 4 * i);
  // LSTM cell (TF1 LSTMCell, gate order i, j, f, o, forget bias 1.0): the split partials in fixed order + bias
  {
    const int u = tid;
    float bz[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) bz[g] = __ldg(a.lstm_b + g * Geo::L + u);
    for (int r = 0; r < kHR; ++r) {
      float hv = 0.f;
      if (r < nr) {
        const int m = row0 + r;
        float z[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          float acc = 0.f;
#pragma unroll
          for (int s = 0; s < kLSplits; ++s) acc += a.zpart[((size_t)s * a.n + m) * Geo::G4 + g * Geo::L + u];
          z[g] = acc + bz[g];
        }
        const float si = sigmoidf_acc(z[0]);
        const float tj = tanhf(z[1]);
        const float sf = sigmoidf_acc(z[2] + 1.0f);
        const float so = sigmoidf_acc(z[3]);
        const float cv = sf * a.c0[(size_t)m * Geo::L + u] + si * tj;
        hv = so * tanhf(cv);
        a.c1[(size_t)m * Geo::L + u] = cv;
        a.h1[(size_t)m * Geo::L + u] = hv;
      }
      sh[r * 256 + u] = hv;
    }
  }
  __syncthreads();
  dense256_relu(sh, a.w1, a.b1, part, shid, tid);    // hid1
  dense256_relu(shid, a.w2, a.b2, part, sh, tid);    // hid2 (over h1, no longer needed)
  const int warp = tid >> 5, lane = tid & 31;
  if (warp >= nr) return;
  const int m = row0 + warp;
  const float* x = sh + warp * 256;
  float logit = -INFINITY;
  if (lane < A) {
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll 4
    for (int k = 0; k < Geo::HID; k += 4) {
      c0 = fmaf(x[k], sw3[k * A + lane], c0);
      c1 = fmaf(x[k + 1], sw3[(k + 1) * A + lane], c1);
      c2 = fmaf(x[k + 2], sw3[(k + 2) * A + lane], c2);
      c3 = fmaf(x[k + 3], sw3[(k + 3) * A + lane], c3);
    }
    logit = ((c0 + c1) + (c2 + c3)) + __ldg(a.b3 + lane);
  }
  const float mx = warp_max(logit);
  const float e = (lane < A) ? expf(logit - mx) : 0.f;
  const float sum = warp_sum(e);
  const float p = e / sum;
  if (lane < A) a.policy[(size_t)m * A + lane] = p;
  // sampling: numpy's RandomState.choice(A, p=policy) for the row's uniform draw (policy_head.cuh)
  float* sp = part + warp * 32;      // the K partials are dead after the second dense layer
  sp[lane] = p;
  __syncwarp();
  const size_t rec_row = (size_t)m * rec.T + *rec.t;
  if (lane < A) rec.mu[rec_row * A + lane] = p;
  if (lane == 0) a.action[m] = rec.action[rec_row] = sample_choice(sp, A, a.uniform, m);
}

// ---- policy_record_step -----------------------------------------------------------------------------------------
// One CTA per row: the frame, previous action, h0 and c0 the act read from the device input block, into step *t of
// the row's trajectory in the recorder's staging.  16-byte copies (frame 28,224 B, h0 / c0 1 KB each).
struct RecordArgs {
  const uint8_t* frames;   // device input block: [n][FRAME]
  const int32_t* pa;       // [n]
  const float* h0;         // [n][256]
  const float* c0;         // [n][256]
  const int32_t* t;        // device word, staged per call
  uint8_t* rec_frames;     // staging [n][T][FRAME]
  int32_t* rec_pa;         // [n][T]
  float* rec_h0;           // [n][T][256]
  float* rec_c0;           // [n][T][256]
  int T;
};
constexpr int kRecThreads = 256;

__global__ void __launch_bounds__(kRecThreads) policy_record_step_kernel(const RecordArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const size_t dst = (size_t)row * a.T + *a.t;
  const uint4* f = reinterpret_cast<const uint4*>(a.frames + (size_t)row * Geo::FRAME);
  uint4* fd = reinterpret_cast<uint4*>(a.rec_frames + dst * Geo::FRAME);
  for (int i = tid; i < Geo::FRAME / 16; i += kRecThreads) fd[i] = f[i];
  if (tid < Geo::L / 4) {
    reinterpret_cast<float4*>(a.rec_h0 + dst * Geo::L)[tid] = reinterpret_cast<const float4*>(a.h0 + (size_t)row * Geo::L)[tid];
  } else if (tid < Geo::L / 2) {
    const int i = tid - Geo::L / 4;
    reinterpret_cast<float4*>(a.rec_c0 + dst * Geo::L)[i] = reinterpret_cast<const float4*>(a.c0 + (size_t)row * Geo::L)[i];
  } else if (tid == Geo::L / 2) {
    a.rec_pa[dst] = a.pa[row];
  }
}

// ---- handle -----------------------------------------------------------------------------------------------------
// device input block of one call with n rows, one contiguous H2D: [frames | previous_action | h0 | c0 | uniform]
struct InLayout {
  size_t frames, pa, h0, c0, u, total;
};
InLayout in_layout(int n) {
  InLayout l;
  size_t off = 0;
  l.frames = off; off = align_up(off + (size_t)n * Geo::FRAME, 256);
  l.pa = off;     off = align_up(off + (size_t)n * 4, 256);
  l.h0 = off;     off = align_up(off + (size_t)n * Geo::L * 4, 256);
  l.c0 = off;     off = align_up(off + (size_t)n * Geo::L * 4, 256);
  l.u = off;      off = align_up(off + (size_t)n * 8, 256);
  l.total = off;
  return l;
}

int set_policy_kernel_attributes() {
  DRL_TRY((set_policy_lstm_attributes<Geo::L, kLSplits>()));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_head_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kHeadSmem));
  DRL_CUDA_CHECK(cudaFuncSetAttribute(policy_head_record_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)kHeadSmem));
  return DRL_OK;
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_policy : PolicyCore {
  ParamLayout pl{};
  // mapped outputs: policy [max_batch][A] | h1 | c1 [max_batch][256] | action
  size_t off_h = 0, off_c = 0, off_act = 0;
};

// the recorder's staging (RecorderCore) is in the queue's field order (TrajField)
struct drl_policy_recorder : RecorderCore {
  drl_policy* policy = nullptr;
};

namespace {

// the engine's mapped outputs of an n-row act
PolicyOutRows mapped_outputs(drl_policy* h) {
  return PolicyOutRows{reinterpret_cast<float*>(h->d_out), reinterpret_cast<float*>(h->d_out + h->off_h),
                       reinterpret_cast<float*>(h->d_out + h->off_c),
                       reinterpret_cast<int32_t*>(h->d_out + h->off_act)};
}

// the kernels of the engine's act of n rows on the device input block d_in, writing `out`; with a recorder, the
// recording head and policy_record_step as well
int enqueue_forward(drl_policy* h, int n, const PolicyOutRows& out, drl_policy_recorder* rec) {
  const InLayout l = in_layout(n);
  const ParamLayout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  const float* h0 = reinterpret_cast<const float*>(h->d_in + l.h0);
  DRL_TRY(conv_forward16(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, h->a1, h->a2, h->a3,
                         h->a1p, h->a2p));
  DRL_TRY((launch_policy_lstm<Geo::L, kLSplits>(s, h->a3, h->table, pa, h0, P + pl.lstm_w, h->zpart, n)));
  HeadArgs a;
  a.zpart = h->zpart;
  a.lstm_b = P + pl.lstm_b;
  a.c0 = reinterpret_cast<const float*>(h->d_in + l.c0);
  a.uniform = reinterpret_cast<const double*>(h->d_in + l.u);
  a.w1 = P + pl.actor1_w; a.b1 = P + pl.actor1_b;
  a.w2 = P + pl.actor2_w; a.b2 = P + pl.actor2_b;
  a.w3 = P + pl.actor3_w; a.b3 = P + pl.actor3_b;
  a.policy = out.policy;
  a.h1 = out.h1;
  a.c1 = out.c1;
  a.action = out.action;
  a.n = n;
  a.A = h->A;
  if (!rec) {
    DRL_CUDA_CHECK((launch_k(policy_head_fused_kernel, cdiv(n, kHR), kHThreads, kHeadSmem, s, a)));
    return DRL_OK;
  }
  HeadRecord hr;
  hr.t = rec->d_t;
  hr.mu = reinterpret_cast<float*>(rec->field(kTrajMu));
  hr.action = reinterpret_cast<int32_t*>(rec->field(kTrajAction));
  hr.T = rec->T;
  DRL_CUDA_CHECK((launch_k(policy_head_record_kernel, cdiv(n, kHR), kHThreads, kHeadSmem, s, a, hr)));
  RecordArgs r;
  r.frames = h->d_in + l.frames;
  r.pa = pa;
  r.h0 = h0;
  r.c0 = a.c0;
  r.t = rec->d_t;
  r.rec_frames = rec->field(kTrajState);
  r.rec_pa = reinterpret_cast<int32_t*>(rec->field(kTrajPa));
  r.rec_h0 = reinterpret_cast<float*>(rec->field(kTrajH));
  r.rec_c0 = reinterpret_cast<float*>(rec->field(kTrajC));
  r.T = rec->T;
  DRL_CUDA_CHECK((launch_k(policy_record_step_kernel, n, kRecThreads, 0, s, r)));
  return DRL_OK;
}

// the engine's act of n rows: the upload of the staged input block, then its kernels
int enqueue_act_impl(drl_policy* h, int n, drl_policy_recorder* rec) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, in_layout(n).total, cudaMemcpyHostToDevice, h->stream));
  return enqueue_forward(h, n, mapped_outputs(h), rec);
}

int enqueue_act(PolicyCore* c, int n) { return enqueue_act_impl(static_cast<drl_policy*>(c), n, nullptr); }

// the recorder's act: the step word, then the recording act of its n rows
int enqueue_record(drl_policy_recorder* r) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(r->d_t, r->h_t, sizeof(int32_t), cudaMemcpyHostToDevice, r->policy->stream));
  return enqueue_act_impl(r->policy, r->n, r);
}

// act's argument checks and the staging of its inputs into h_in (the caller holds the engine's lock)
int stage_act(drl_policy* h, int n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
              const float* c_in, const double* uniform, const int32_t* action) {
  DRL_TRY(policy_check_n(h, n, state && previous_action && h_in && c_in));
  if (action && !uniform) { set_error("act: `action` needs `uniform` (one draw in [0, 1) per row)"); return DRL_ERR_INVALID; }
  DRL_TRY(policy_check_actions(h, n, previous_action, nullptr));
  // the previous call has completed (this entry point is synchronous): the staging block is free
  const InLayout l = in_layout(n);
  memcpy(h->h_in + l.frames, state, (size_t)n * Geo::FRAME);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
  memcpy(h->h_in + l.h0, h_in, (size_t)n * Geo::L * 4);
  memcpy(h->h_in + l.c0, c_in, (size_t)n * Geo::L * 4);
  if (uniform) memcpy(h->h_in + l.u, uniform, (size_t)n * 8);
  else memset(h->h_in + l.u, 0, (size_t)n * 8);
  return DRL_OK;
}

void copy_act_outputs(const drl_policy* h, int n, int32_t* action, float* policy, float* h_out, float* c_out) {
  if (policy) memcpy(policy, h->h_out, (size_t)n * h->A * 4);
  if (h_out) memcpy(h_out, h->h_out + h->off_h, (size_t)n * Geo::L * 4);
  if (c_out) memcpy(c_out, h->h_out + h->off_c, (size_t)n * Geo::L * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
}

}  // namespace

namespace drl {

PolicyCore* policy_core_of(drl_policy* h) { return h; }

PolicyInRows policy_input_rows(drl_policy* h, int n) {
  const InLayout l = in_layout(n);
  return PolicyInRows{h->d_in + l.frames, reinterpret_cast<int32_t*>(h->d_in + l.pa),
                      reinterpret_cast<float*>(h->d_in + l.h0), reinterpret_cast<float*>(h->d_in + l.c0),
                      reinterpret_cast<double*>(h->d_in + l.u)};
}

int policy_enqueue_forward(drl_policy* h, int n, const PolicyOutRows& out) {
  return enqueue_forward(h, n, out, nullptr);
}

}  // namespace drl

extern "C" {

int drl_policy_create(const drl_policy_config* cfg, drl_policy** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->max_batch < 1 || cfg->max_batch > kMaxPolicyRows) {
    set_error("max_batch must be in [1, %d] (got %d)", kMaxPolicyRows, cfg->max_batch);
    return DRL_ERR_INVALID;
  }
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || cfg->channels != Geo::IC) {
    set_error("only the reference input geometry 84x84x4 is supported (got %dx%dx%d)", cfg->height, cfg->width,
              cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->lstm_size != Geo::L) { set_error("only lstm_size 256 is supported (got %d)", cfg->lstm_size); return DRL_ERR_INVALID; }
  if (cfg->num_action < 2 || cfg->num_action > kMaxA) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  DRL_TRY(policy_check_device(cfg->device));
  NvtxRange nv("drl:policy_create");
  drl_policy* h = new drl_policy();
  h->device = cfg->device;
  h->max_batch = cfg->max_batch;
  h->A = cfg->num_action;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->splits = kLSplits;
  h->zpart_cols = Geo::G4;
  h->pl.init(h->A);
  h->layout = &h->pl;
  h->enqueue_act = enqueue_act;
  h->conv_images = [](cudaStream_t s, const TrunkLayout& pl, const float* P, uint8_t* img_conv2, uint8_t* img_conv3) {
    return conv_images16(s, static_cast<const ParamLayout&>(pl), P, img_conv2, img_conv3);
  };
  const size_t MB = cfg->max_batch;
  h->off_h = align_up(MB * kMaxA * 4, 256);
  h->off_c = h->off_h + align_up(MB * Geo::L * 4, 256);
  h->off_act = h->off_c + align_up(MB * Geo::L * 4, 256);
  const size_t out_bytes = h->off_act + align_up(MB * 4, 256);
  const int rc = policy_core_init(h, set_policy_kernel_attributes, kLSplits * MB * Geo::G4, in_layout(MB).total,
                                  out_bytes);
  if (rc != DRL_OK) { delete h; return rc; }
  *out = h;
  return DRL_OK;
}

int drl_policy_destroy(drl_policy* h) { return policy_destroy(h); }
int drl_policy_param_count(const drl_policy* h, int64_t* n) { return policy_param_count(h, kName, n); }
int drl_policy_set_params(drl_policy* h, const float* host_flat, int64_t n) {
  return policy_set_params(h, kName, host_flat, n);
}
int drl_policy_get_params(drl_policy* h, float* host_flat, int64_t n) {
  return policy_get_params(h, kName, host_flat, n);
}
int drl_policy_sync_from_learner(drl_policy* h, drl_learner* learner) {
  return policy_sync(h, kName, learner, [&] {
    return impala_params_snapshot(learner, h->device, h->A, h->stream, h->params, h->ev_ready, h->ev_copied);
  });
}
int drl_policy_last_act_ms(drl_policy* h, float* ms) { return policy_last_act_ms(h, kName, ms); }
int drl_policy_read_buffer(drl_policy* h, const char* name, float* host_dst, int64_t n) {
  return policy_read_buffer(h, kName, name, host_dst, n);
}
int drl_policy_buffer_dims(drl_policy* h, int32_t* out) { return policy_buffer_dims(h, kName, out); }

int drl_policy_act(drl_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
                   const float* c_in, const double* uniform, int32_t* action, float* policy, float* h_out,
                   float* c_out) {
  DRL_TRY(policy_check(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(stage_act(h, n, state, previous_action, h_in, c_in, uniform, action));
  NvtxRange nv("drl:policy_act");
  DRL_TRY(policy_run_act(h, n));
  copy_act_outputs(h, n, action, policy, h_out, c_out);
  return DRL_OK;
}

// ---- recorder ---------------------------------------------------------------------------------------------------
int drl_policy_recorder_create(drl_policy* h, drl_traj_queue* q, int32_t n, drl_policy_recorder** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  DRL_TRY(policy_check(h, kName));
  if (!q) { set_error("null trajectory queue handle"); return DRL_ERR_INVALID; }
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > h->max_batch) {
    set_error("recorder: n must be in [1, %d] (the engine's max_batch; got %d)", h->max_batch, n);
    return DRL_ERR_INVALID;
  }
  if (q->device != h->device) {
    set_error("recorder: the queue is on device %d, the policy on device %d", q->device, h->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != h->A) { set_error("recorder: the queue has num_action %d, the policy %d", q->A, h->A); return DRL_ERR_INVALID; }
  if (q->H != Geo::IH || q->W != Geo::IW || q->C != Geo::IC || q->L != Geo::L) {
    set_error("recorder: the queue stores %dx%dx%d frames and lstm %d, the policy takes %dx%dx%d and %d", q->H, q->W,
              q->C, q->L, Geo::IH, Geo::IW, Geo::IC, Geo::L);
    return DRL_ERR_INVALID;
  }
  if (n > traj_queue_max_rows(q)) {
    set_error("recorder: %d rows per commit can never fit in the queue (at most %d)", n, traj_queue_max_rows(q));
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:policy_recorder_create");
  drl_policy_recorder* r = new drl_policy_recorder();
  r->engine = r->policy = h;
  r->q = q;
  r->n = n;
  r->T = q->T;
  r->f_reward = kTrajReward;
  r->f_done = kTrajDone;
  const int rc = recorder_core_init(r);
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    recorder_core_release(r);
    delete r;
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = r;
  return DRL_OK;
}

int drl_policy_recorder_destroy(drl_policy_recorder* r) { return recorder_destroy(r); }

int drl_policy_recorder_act(drl_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                            const float* h_in, const float* c_in, const double* uniform, int32_t* action,
                            float* policy, float* h_out, float* c_out) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  drl_policy* h = r->policy;
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(recorder_check_step(r));
  if (!uniform) { set_error("recorder act: `uniform` is required (the recorded actions are the sampled ones)"); return DRL_ERR_INVALID; }
  DRL_TRY(stage_act(h, r->n, state, previous_action, h_in, c_in, uniform, action));
  NvtxRange nv("drl:policy_recorder_act");
  DRL_TRY(recorder_run_act(r, [r] { return enqueue_record(r); }));
  copy_act_outputs(h, r->n, action, policy, h_out, c_out);
  return DRL_OK;
}

int drl_policy_recorder_commit(drl_policy_recorder* r, const float* reward, const uint8_t* done, int32_t timeout_ms) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  return recorder_commit(r, reward, done, timeout_ms);
}

int drl_policy_recorder_reset(drl_policy_recorder* r) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  return recorder_reset(r);
}

}  // extern "C"
