// r2d2_policy.cu -- the R2D2 policy engine behind drl_r2d2_policy_* (include/drl_b200.h): the actor side of
// train_r2d2.py:167-251.  A forward-only handle that runs network() of the main scope (model/r2d2_lstm.py:28-53) for
// n <= 64 environments per call and applies the action rule of Agent.get_action (agent/r2d2.py:171-191) on the GPU,
// with the explore decision and the random action drawn on the host.
//
// One call = one H2D of the staged inputs + 5 kernels on the engine's own stream:
//   conv1 / conv2 / conv3   the R2D2 learner's math-mode-2 kernels and configurations (layer_defs.cuh: conv_forward_tf32)
//   policy_lstm_fwd         z = [a3 | table[pa] | h0] W_lstm as a skinny split-K FP32-FFMA GEMM (K = 3456, N = 256,
//                           policy_lstm.cuh): 2 column chunks x kR2Splits K splits
//   r2d2_policy_head        split-K sum + bias + gates (c', h'), q1 = relu(h' W_q1 + b), q = (value + b_v) - mean,
//                           first-maximum argmax and the explore override; writes q, h', c', action and q[action]
//                           straight into mapped pinned memory (no D2H node)
// Both new kernels sum in a fixed order without atomics: eager and graph replays, and repeated calls, are bitwise equal.
// The act enqueues two halves: the H2D of its pinned input block, then the kernels on the device input block
// (r2d2_policy_enqueue_forward), which the R2D2 policy server (r2d2_policy_server.cu) runs on input rows its own kernel
// fills.
//
// A recorder (drl_r2d2_policy_recorder_*, DESIGN.md section 13) binds the engine to a device R2D2 sequence queue
// (traj_queue.cuh, queue_recorder.cuh).  Its act is the engine's act with r2d2_policy_head_record in place of
// r2d2_policy_head (the same head that also writes the chosen action into the recorder's staging) plus
// r2d2_record_step (frames and previous action of the device input block, and at step 0 h0 and c0, into the staging);
// the step t reaches both through a device word staged per call, so one graph per recorder replays every step.
#include <string.h>

#include "policy_core.cuh"
#include "policy_lstm.cuh"
#include "queue_recorder.cuh"
#include "r2d2_defs.cuh"

namespace drl {
namespace {

constexpr const char* kName = "r2d2 policy";
constexpr int kMaxR2PolicyRows = 64;
constexpr int kR2MaxA = 32;

// ---- policy_lstm_fwd (policy_lstm.cuh) --------------------------------------------------------------------------
// grid (256 / kLN column chunks) x (kR2Splits K splits) = 2 x 48 = 96 CTAs: one wave on the 132 SMs of an H100, each
// streaming its 72 x 128 fp32 slab of W (36 KB) once.
constexpr int kR2Splits = 48;

// ---- r2d2_policy_head -------------------------------------------------------------------------------------------
// One CTA per row, 256 threads.  Thread j sums gate column j over the splits in index order, adds the bias and applies
// its gate's nonlinearity (TF1 LSTMCell: i, j, f, o, forget bias 1.0); threads < 64 form c' and h'.  q1: thread u < 128
// owns output u (K = 64 in four interleaved chains added in fixed order).  value / mean: the lane layout of
// r2d2_out_kernel (lane owns q1[lane + 32 i], warp_sum, q = (v + b_v) - mean); warp w computes the actions a = w mod 8.
struct R2HeadArgs {
  const float* zpart;       // [kR2Splits][n][256]
  const float* lstm_b;      // [256]
  const float* c0;          // [n][64]
  const int32_t* explore;   // [n]: -1 greedy, otherwise the action
  const float *q1_w, *q1_b, *value_w, *value_b, *mean_w, *mean_b;
  float* q;                 // mapped outputs: [n][A]
  float* h1;                // [n][64]
  float* c1;                // [n][64]
  int32_t* action;          // [n]
  float* q_action;          // [n]
  int n, A;
};

__global__ void __launch_bounds__(kR2G, 1) r2d2_policy_head_kernel(const R2HeadArgs a) {
  kernel_prologue();
  __shared__ float sg[kR2G];
  __shared__ __align__(16) float sh[kR2L];
  __shared__ float sq1[kR2H];
  __shared__ float sq[kR2MaxA];
  const int m = blockIdx.x, j = threadIdx.x;
  {
    float z = 0.f;
#pragma unroll 8
    for (int s = 0; s < kR2Splits; ++s) z += a.zpart[((size_t)s * a.n + m) * kR2G + j];
    const float pre = z + __ldg(a.lstm_b + j);
    const int gate = j / kR2L;
    sg[j] = (gate == 1) ? tanhf(pre) : sigmoidf_acc(gate == 2 ? pre + 1.0f : pre);
  }
  __syncthreads();
  if (j < kR2L) {
    const float si = sg[j], tj = sg[kR2L + j], sf = sg[2 * kR2L + j], so = sg[3 * kR2L + j];
    const float c = sf * a.c0[(size_t)m * kR2L + j] + si * tj;
    const float h = so * tanhf(c);
    a.c1[(size_t)m * kR2L + j] = c;
    a.h1[(size_t)m * kR2L + j] = h;
    sh[j] = h;
  }
  __syncthreads();
  if (j < kR2H) {
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
    for (int k = 0; k < kR2L; k += 4) {
      const float4 h4 = *reinterpret_cast<const float4*>(sh + k);
      c0 = fmaf(h4.x, __ldg(a.q1_w + (size_t)k * kR2H + j), c0);
      c1 = fmaf(h4.y, __ldg(a.q1_w + (size_t)(k + 1) * kR2H + j), c1);
      c2 = fmaf(h4.z, __ldg(a.q1_w + (size_t)(k + 2) * kR2H + j), c2);
      c3 = fmaf(h4.w, __ldg(a.q1_w + (size_t)(k + 3) * kR2H + j), c3);
    }
    sq1[j] = fmaxf(((c0 + c1) + (c2 + c3)) + __ldg(a.q1_b + j), 0.f);
  }
  __syncthreads();
  const int warp = j >> 5, lane = j & 31, A = a.A;
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = sq1[lane + 32 * i];
  float mean = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) mean = fmaf(x[i], __ldg(a.mean_w + lane + 32 * i), mean);
  mean = warp_sum(mean) + __ldg(a.mean_b);
  for (int act = warp; act < A; act += kR2G / 32) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) v = fmaf(x[i], __ldg(a.value_w + (size_t)(lane + 32 * i) * A + act), v);
    v = warp_sum(v);
    if (lane == 0) {
      const float qv = (v + __ldg(a.value_b + act)) - mean;
      sq[act] = qv;
      a.q[(size_t)m * A + act] = qv;
    }
  }
  __syncthreads();
  if (j == 0) {
    // np.argmax: the first maximum
    float best = sq[0];
    int arg = 0;
    for (int k = 1; k < A; ++k) {
      if (sq[k] > best) { best = sq[k]; arg = k; }
    }
    const int e = a.explore[m];
    const int act = e >= 0 ? e : arg;
    a.action[m] = act;
    a.q_action[m] = sq[act];
  }
}

// what the recording head writes besides R2HeadArgs' outputs: the action of step *t of rows 0..n-1
struct R2HeadRecord {
  const int32_t* t;         // device word, staged per call
  int32_t* action;          // [n][S]
  int S;
};

// The recording head: r2d2_policy_head_kernel, plus each row's chosen action (the explore override included) written
// into a recorder's staging at step *rec.t.  A separate copy, so that r2d2_policy_head_kernel and R2HeadArgs keep their
// source and the code nvcc generates for them.
__global__ void __launch_bounds__(kR2G, 1) r2d2_policy_head_record_kernel(const R2HeadArgs a,
                                                                                  const R2HeadRecord rec) {
  kernel_prologue();
  __shared__ float sg[kR2G];
  __shared__ __align__(16) float sh[kR2L];
  __shared__ float sq1[kR2H];
  __shared__ float sq[kR2MaxA];
  const int m = blockIdx.x, j = threadIdx.x;
  {
    float z = 0.f;
#pragma unroll 8
    for (int s = 0; s < kR2Splits; ++s) z += a.zpart[((size_t)s * a.n + m) * kR2G + j];
    const float pre = z + __ldg(a.lstm_b + j);
    const int gate = j / kR2L;
    sg[j] = (gate == 1) ? tanhf(pre) : sigmoidf_acc(gate == 2 ? pre + 1.0f : pre);
  }
  __syncthreads();
  if (j < kR2L) {
    const float si = sg[j], tj = sg[kR2L + j], sf = sg[2 * kR2L + j], so = sg[3 * kR2L + j];
    const float c = sf * a.c0[(size_t)m * kR2L + j] + si * tj;
    const float h = so * tanhf(c);
    a.c1[(size_t)m * kR2L + j] = c;
    a.h1[(size_t)m * kR2L + j] = h;
    sh[j] = h;
  }
  __syncthreads();
  if (j < kR2H) {
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
    for (int k = 0; k < kR2L; k += 4) {
      const float4 h4 = *reinterpret_cast<const float4*>(sh + k);
      c0 = fmaf(h4.x, __ldg(a.q1_w + (size_t)k * kR2H + j), c0);
      c1 = fmaf(h4.y, __ldg(a.q1_w + (size_t)(k + 1) * kR2H + j), c1);
      c2 = fmaf(h4.z, __ldg(a.q1_w + (size_t)(k + 2) * kR2H + j), c2);
      c3 = fmaf(h4.w, __ldg(a.q1_w + (size_t)(k + 3) * kR2H + j), c3);
    }
    sq1[j] = fmaxf(((c0 + c1) + (c2 + c3)) + __ldg(a.q1_b + j), 0.f);
  }
  __syncthreads();
  const int warp = j >> 5, lane = j & 31, A = a.A;
  float x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = sq1[lane + 32 * i];
  float mean = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) mean = fmaf(x[i], __ldg(a.mean_w + lane + 32 * i), mean);
  mean = warp_sum(mean) + __ldg(a.mean_b);
  for (int act = warp; act < A; act += kR2G / 32) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) v = fmaf(x[i], __ldg(a.value_w + (size_t)(lane + 32 * i) * A + act), v);
    v = warp_sum(v);
    if (lane == 0) {
      const float qv = (v + __ldg(a.value_b + act)) - mean;
      sq[act] = qv;
      a.q[(size_t)m * A + act] = qv;
    }
  }
  __syncthreads();
  if (j == 0) {
    // np.argmax: the first maximum
    float best = sq[0];
    int arg = 0;
    for (int k = 1; k < A; ++k) {
      if (sq[k] > best) { best = sq[k]; arg = k; }
    }
    const int e = a.explore[m];
    const int act = e >= 0 ? e : arg;
    a.action[m] = rec.action[(size_t)m * rec.S + *rec.t] = act;
    a.q_action[m] = sq[act];
  }
}

// ---- r2d2_record_step -------------------------------------------------------------------------------------------
// One CTA per row: the frame and previous action the act read from the device input block into step *t of the row's
// sequence in the recorder's staging, and at step 0 the row's h0 and c0 (a record keeps the state of step 0 only, the
// (h, c) carried in from the previous unroll).  16-byte copies (frame 7,056 or 28,224 B, h0 / c0 256 B each).
struct R2RecordArgs {
  const uint8_t* frames;    // device input block: [n][frame]
  const int32_t* pa;        // [n]
  const float* h0;          // [n][64]
  const float* c0;          // [n][64]
  const int32_t* t;         // device word, staged per call
  uint8_t* rec_frames;      // staging [n][S][frame]
  int32_t* rec_pa;          // [n][S]
  float* rec_h0;            // [n][64]
  float* rec_c0;            // [n][64]
  int S, frame16;           // frame16: 16-byte vectors per frame
};
constexpr int kR2RecThreads = 256;

__global__ void __launch_bounds__(kR2RecThreads) r2d2_record_step_kernel(const R2RecordArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x, t = *a.t;
  const size_t dst = (size_t)row * a.S + t;
  const uint4* f = reinterpret_cast<const uint4*>(a.frames) + (size_t)row * a.frame16;
  uint4* fd = reinterpret_cast<uint4*>(a.rec_frames) + dst * a.frame16;
  for (int i = tid; i < a.frame16; i += kR2RecThreads) fd[i] = f[i];
  if (tid == 0) a.rec_pa[dst] = a.pa[row];
  if (t == 0 && tid < 2 * (kR2L / 4)) {
    const int k = tid % (kR2L / 4);
    const float* src = tid < kR2L / 4 ? a.h0 : a.c0;
    float* d = tid < kR2L / 4 ? a.rec_h0 : a.rec_c0;
    reinterpret_cast<float4*>(d + (size_t)row * kR2L)[k] = reinterpret_cast<const float4*>(src + (size_t)row * kR2L)[k];
  }
}

// ---- handle -----------------------------------------------------------------------------------------------------
// device input block of one call with n rows, one contiguous H2D: [frames | previous_action | h0 | c0 | explore]
struct R2InLayout {
  size_t frames, pa, h0, c0, explore, total;
};
R2InLayout r2_in_layout(int n, size_t frame) {
  R2InLayout l;
  size_t off = 0;
  l.frames = off;  off = align_up(off + (size_t)n * frame, 256);
  l.pa = off;      off = align_up(off + (size_t)n * 4, 256);
  l.h0 = off;      off = align_up(off + (size_t)n * kR2L * 4, 256);
  l.c0 = off;      off = align_up(off + (size_t)n * kR2L * 4, 256);
  l.explore = off; off = align_up(off + (size_t)n * 4, 256);
  l.total = off;
  return l;
}

int set_r2_policy_kernel_attributes() { return set_policy_lstm_attributes<kR2L, kR2Splits>(); }

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_r2d2_policy : PolicyCore {
  R2Layout pl{};
  size_t frame = 0;
  // mapped outputs: q [max_batch][A] | h' | c' [max_batch][64] | action | q_action
  size_t off_h = 0, off_c = 0, off_act = 0, off_qa = 0;
};

// the recorder's staging (RecorderCore) is in the queue's field order (R2QueueField)
struct drl_r2d2_policy_recorder : RecorderCore {
  drl_r2d2_policy* policy = nullptr;
};

namespace {

// the engine's mapped outputs of an n-row act
R2PolicyOutRows mapped_outputs(drl_r2d2_policy* h) {
  return R2PolicyOutRows{reinterpret_cast<float*>(h->d_out), reinterpret_cast<float*>(h->d_out + h->off_h),
                         reinterpret_cast<float*>(h->d_out + h->off_c),
                         reinterpret_cast<int32_t*>(h->d_out + h->off_act),
                         reinterpret_cast<float*>(h->d_out + h->off_qa)};
}

// the kernels of the engine's act of n rows on the device input block d_in, writing `out`; with a recorder, the
// recording head and r2d2_record_step as well
int enqueue_forward(drl_r2d2_policy* h, int n, const R2PolicyOutRows& out, drl_r2d2_policy_recorder* rec) {
  const R2InLayout l = r2_in_layout(n, h->frame);
  const R2Layout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  const float* h0 = reinterpret_cast<const float*>(h->d_in + l.h0);
  DRL_TRY(policy_conv_forward_tf32(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, h->a1, h->a2, h->a3));
  DRL_TRY((launch_policy_lstm<kR2L, kR2Splits>(s, h->a3, h->table, pa, h0, P + pl.lstm_w, h->zpart, n)));
  R2HeadArgs a;
  a.zpart = h->zpart;
  a.lstm_b = P + pl.lstm_b;
  a.c0 = reinterpret_cast<const float*>(h->d_in + l.c0);
  a.explore = reinterpret_cast<const int32_t*>(h->d_in + l.explore);
  a.q1_w = P + pl.q1_w; a.q1_b = P + pl.q1_b;
  a.value_w = P + pl.value_w; a.value_b = P + pl.value_b;
  a.mean_w = P + pl.mean_w; a.mean_b = P + pl.mean_b;
  a.q = out.q;
  a.h1 = out.h1;
  a.c1 = out.c1;
  a.action = out.action;
  a.q_action = out.q_action;
  a.n = n;
  a.A = h->A;
  if (!rec) {
    DRL_CUDA_CHECK((launch_k(r2d2_policy_head_kernel, n, kR2G, 0, s, a)));
    return DRL_OK;
  }
  R2HeadRecord hr;
  hr.t = rec->d_t;
  hr.action = reinterpret_cast<int32_t*>(rec->field(kR2QAction));
  hr.S = rec->T;
  DRL_CUDA_CHECK((launch_k(r2d2_policy_head_record_kernel, n, kR2G, 0, s, a, hr)));
  R2RecordArgs r;
  r.frames = h->d_in + l.frames;
  r.pa = pa;
  r.h0 = h0;
  r.c0 = a.c0;
  r.t = rec->d_t;
  r.rec_frames = rec->field(kR2QFrames);
  r.rec_pa = reinterpret_cast<int32_t*>(rec->field(kR2QPa));
  r.rec_h0 = reinterpret_cast<float*>(rec->field(kR2QH));
  r.rec_c0 = reinterpret_cast<float*>(rec->field(kR2QC));
  r.S = rec->T;
  r.frame16 = (int)(h->frame / 16);
  DRL_CUDA_CHECK((launch_k(r2d2_record_step_kernel, n, kR2RecThreads, 0, s, r)));
  return DRL_OK;
}

// the engine's act of n rows: the upload of the staged input block, then its kernels
int enqueue_act_impl(drl_r2d2_policy* h, int n, drl_r2d2_policy_recorder* rec) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, r2_in_layout(n, h->frame).total, cudaMemcpyHostToDevice, h->stream));
  return enqueue_forward(h, n, mapped_outputs(h), rec);
}

int enqueue_act(PolicyCore* c, int n) { return enqueue_act_impl(static_cast<drl_r2d2_policy*>(c), n, nullptr); }

// the recorder's act: the step word, then the recording act of its n rows
int enqueue_record(drl_r2d2_policy_recorder* r) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(r->d_t, r->h_t, sizeof(int32_t), cudaMemcpyHostToDevice, r->policy->stream));
  return enqueue_act_impl(r->policy, r->n, r);
}

// act's argument checks and the staging of its inputs into h_in (the caller holds the engine's lock)
int stage_act(drl_r2d2_policy* h, int n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
              const float* c_in, const int32_t* explore_action) {
  DRL_TRY(policy_check_n(h, n, state && previous_action && h_in && c_in));
  DRL_TRY(policy_check_actions(h, n, previous_action, explore_action));
  // the previous call has completed (this entry point is synchronous): the staging block is free
  const R2InLayout l = r2_in_layout(n, h->frame);
  memcpy(h->h_in + l.frames, state, (size_t)n * h->frame);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
  memcpy(h->h_in + l.h0, h_in, (size_t)n * kR2L * 4);
  memcpy(h->h_in + l.c0, c_in, (size_t)n * kR2L * 4);
  policy_stage_explore(h->h_in + l.explore, explore_action, n);
  return DRL_OK;
}

void copy_act_outputs(const drl_r2d2_policy* h, int n, int32_t* action, float* q, float* q_action, float* h_out,
                      float* c_out) {
  if (q) memcpy(q, h->h_out, (size_t)n * h->A * 4);
  if (h_out) memcpy(h_out, h->h_out + h->off_h, (size_t)n * kR2L * 4);
  if (c_out) memcpy(c_out, h->h_out + h->off_c, (size_t)n * kR2L * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
  if (q_action) memcpy(q_action, h->h_out + h->off_qa, (size_t)n * 4);
}

}  // namespace

namespace drl {

PolicyCore* r2d2_policy_core_of(drl_r2d2_policy* h) { return h; }
int r2d2_policy_channels(const drl_r2d2_policy* h) { return h->pl.C; }

R2PolicyInRows r2d2_policy_input_rows(drl_r2d2_policy* h, int n) {
  const R2InLayout l = r2_in_layout(n, h->frame);
  return R2PolicyInRows{h->d_in + l.frames, reinterpret_cast<int32_t*>(h->d_in + l.pa),
                        reinterpret_cast<float*>(h->d_in + l.h0), reinterpret_cast<float*>(h->d_in + l.c0),
                        reinterpret_cast<int32_t*>(h->d_in + l.explore)};
}

int r2d2_policy_enqueue_forward(drl_r2d2_policy* h, int n, const R2PolicyOutRows& out) {
  return enqueue_forward(h, n, out, nullptr);
}

}  // namespace drl

extern "C" {

int drl_r2d2_policy_create(const drl_r2d2_policy_config* cfg, drl_r2d2_policy** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->max_batch < 1 || cfg->max_batch > kMaxR2PolicyRows) {
    set_error("max_batch must be in [1, %d] (got %d)", kMaxR2PolicyRows, cfg->max_batch);
    return DRL_ERR_INVALID;
  }
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || (cfg->channels != 1 && cfg->channels != 4)) {
    set_error("only 84x84x1 and 84x84x4 frames are supported (got %dx%dx%d)", cfg->height, cfg->width, cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->lstm_size != kR2L) { set_error("only lstm_size %d is supported (got %d)", kR2L, cfg->lstm_size); return DRL_ERR_INVALID; }
  if (cfg->num_action < 2 || cfg->num_action > kR2MaxA) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  DRL_TRY(policy_check_device(cfg->device));
  NvtxRange nv("drl:r2d2_policy_create");
  drl_r2d2_policy* h = new drl_r2d2_policy();
  h->device = cfg->device;
  h->max_batch = cfg->max_batch;
  h->A = cfg->num_action;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->splits = kR2Splits;
  h->zpart_cols = kR2G;
  h->frame = (size_t)Geo::IH * Geo::IW * cfg->channels;
  h->pl.init(h->A, cfg->channels);
  h->layout = &h->pl;
  h->enqueue_act = enqueue_act;
  h->conv_images = policy_conv_images_tf32;
  const size_t MB = cfg->max_batch;
  h->off_h = align_up(MB * kR2MaxA * 4, 256);
  h->off_c = h->off_h + align_up(MB * kR2L * 4, 256);
  h->off_act = h->off_c + align_up(MB * kR2L * 4, 256);
  h->off_qa = h->off_act + align_up(MB * 4, 256);
  const size_t out_bytes = h->off_qa + align_up(MB * 4, 256);
  const int rc = policy_core_init(h, set_r2_policy_kernel_attributes, kR2Splits * MB * kR2G,
                                  r2_in_layout(MB, h->frame).total, out_bytes);
  if (rc != DRL_OK) { delete h; return rc; }
  *out = h;
  return DRL_OK;
}

int drl_r2d2_policy_destroy(drl_r2d2_policy* h) { return policy_destroy(h); }
int drl_r2d2_policy_param_count(const drl_r2d2_policy* h, int64_t* n) { return policy_param_count(h, kName, n); }
int drl_r2d2_policy_set_params(drl_r2d2_policy* h, const float* host_flat, int64_t n) {
  return policy_set_params(h, kName, host_flat, n);
}
int drl_r2d2_policy_get_params(drl_r2d2_policy* h, float* host_flat, int64_t n) {
  return policy_get_params(h, kName, host_flat, n);
}
int drl_r2d2_policy_sync_from_learner(drl_r2d2_policy* h, drl_r2d2* learner) {
  return policy_sync(h, kName, learner, [&] {
    return r2d2_params_snapshot(learner, h->device, h->A, h->pl.C, h->stream, h->params, h->ev_ready, h->ev_copied);
  });
}
int drl_r2d2_policy_last_act_ms(drl_r2d2_policy* h, float* ms) { return policy_last_act_ms(h, kName, ms); }
int drl_r2d2_policy_read_buffer(drl_r2d2_policy* h, const char* name, float* host_dst, int64_t n) {
  return policy_read_buffer(h, kName, name, host_dst, n);
}
int drl_r2d2_policy_buffer_dims(drl_r2d2_policy* h, int32_t* out) { return policy_buffer_dims(h, kName, out); }

int drl_r2d2_policy_act(drl_r2d2_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const float* h_in, const float* c_in, const int32_t* explore_action, int32_t* action, float* q,
                        float* q_action, float* h_out, float* c_out) {
  DRL_TRY(policy_check(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(stage_act(h, n, state, previous_action, h_in, c_in, explore_action));
  NvtxRange nv("drl:r2d2_policy_act");
  DRL_TRY(policy_run_act(h, n));
  copy_act_outputs(h, n, action, q, q_action, h_out, c_out);
  return DRL_OK;
}

// ---- recorder ---------------------------------------------------------------------------------------------------
int drl_r2d2_policy_recorder_create(drl_r2d2_policy* h, drl_r2d2_queue* q, int32_t n, drl_r2d2_policy_recorder** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  DRL_TRY(policy_check(h, kName));
  if (!q) { set_error("null r2d2 queue handle"); return DRL_ERR_INVALID; }
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
  if (q->C != h->pl.C) {
    set_error("recorder: the queue stores 84x84x%d frames, the policy takes 84x84x%d", q->C, h->pl.C);
    return DRL_ERR_INVALID;
  }
  if (n > traj_queue_max_rows(q)) {
    set_error("recorder: %d rows per commit can never fit in the queue (at most %d)", n, traj_queue_max_rows(q));
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:r2d2_policy_recorder_create");
  drl_r2d2_policy_recorder* r = new drl_r2d2_policy_recorder();
  r->engine = r->policy = h;
  r->q = q;
  r->n = n;
  r->T = q->S;
  r->f_reward = kR2QReward;
  r->f_done = kR2QDone;
  r->last_step = "S-1";
  r->commit_range = "drl:r2d2_policy_recorder_commit";
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

int drl_r2d2_policy_recorder_destroy(drl_r2d2_policy_recorder* r) { return recorder_destroy(r); }

int drl_r2d2_policy_recorder_act(drl_r2d2_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                                 const float* h_in, const float* c_in, const int32_t* explore_action, int32_t* action,
                                 float* q, float* q_action, float* h_out, float* c_out) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  drl_r2d2_policy* h = r->policy;
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(recorder_check_step(r));
  DRL_TRY(stage_act(h, r->n, state, previous_action, h_in, c_in, explore_action));
  NvtxRange nv("drl:r2d2_policy_recorder_act");
  DRL_TRY(recorder_run_act(r, [r] { return enqueue_record(r); }));
  copy_act_outputs(h, r->n, action, q, q_action, h_out, c_out);
  return DRL_OK;
}

int drl_r2d2_policy_recorder_commit(drl_r2d2_policy_recorder* r, const float* reward, const uint8_t* done,
                                    int32_t timeout_ms) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  return recorder_commit(r, reward, done, timeout_ms);
}

int drl_r2d2_policy_recorder_reset(drl_r2d2_policy_recorder* r) {
  if (!r) { set_error("null recorder handle"); return DRL_ERR_INVALID; }
  return recorder_reset(r);
}

}  // extern "C"
