// r2d2_policy.cu -- the R2D2 policy engine behind drl_r2d2_policy_* (include/drl_b200.h): the actor side of
// train_r2d2.py:167-251.  A forward-only handle that runs network() of the main scope (model/r2d2_lstm.py:28-53) for
// n <= 64 environments per call and applies the action rule of Agent.get_action (agent/r2d2.py:171-191) on the GPU,
// with the explore decision and the random action drawn on the host.
//
// One call = one H2D of the staged inputs + 5 kernels on the engine's own stream:
//   conv1 / conv2 / conv3   the R2D2 learner's math-mode-2 kernels and configurations (r2d2.cu: r2_conv_forward)
//   policy_lstm_fwd         z = [a3 | table[pa] | h0] W_lstm as a skinny split-K FP32-FFMA GEMM (K = 3456, N = 256,
//                           policy_lstm.cuh): 2 column chunks x kR2Splits K splits
//   r2d2_policy_head        split-K sum + bias + gates (c', h'), q1 = relu(h' W_q1 + b), q = (value + b_v) - mean,
//                           first-maximum argmax and the explore override; writes q, h', c', action and q[action]
//                           straight into mapped pinned memory (no D2H node)
// Both new kernels sum in a fixed order without atomics: eager and graph replays, and repeated calls, are bitwise equal.
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "policy_lstm.cuh"
#include "r2d2_defs.cuh"

namespace drl {
namespace {

struct R2PolicyNvtx {
  explicit R2PolicyNvtx(const char* name) { nvtxRangePushA(name); }
  ~R2PolicyNvtx() { nvtxRangePop(); }
};

constexpr int kMaxR2PolicyRows = 64;
constexpr int kR2MaxA = 32;
constexpr int kR2ConvMode = 2;     // the learner's default math mode (wgmma 3xTF32 convolutions on weight images)

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

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_r2d2_policy {
  drl_r2d2_policy_config cfg{};
  int A = 0;
  size_t frame = 0;
  R2Layout pl{};
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_ready = nullptr, ev_copied = nullptr;   // learner -> policy and policy -> learner edges of a sync
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;     // device time of the last act
  bool timed = false;
  float* params = nullptr;       // padded main-scope vector (learner layout)
  uint8_t* img_conv2 = nullptr;  // conv2 / conv3 forward weight images (math mode 2)
  uint8_t* img_conv3 = nullptr;
  float* e1 = nullptr;           // [A,256] relu(emb1), scratch of emb_forward
  float* table = nullptr;        // [A,256] action-embedding table (depends on the parameters only)
  float *a1 = nullptr, *a2 = nullptr, *a3 = nullptr;
  float* zpart = nullptr;        // [kR2Splits][max_batch][256]
  uint8_t* d_in = nullptr;       // device input block (r2_in_layout)
  uint8_t* h_in = nullptr;       // pinned staging of the same block
  uint8_t* h_out = nullptr;      // mapped pinned outputs: q [max_batch][A] | h' | c' [max_batch][64] | action | q_action
  uint8_t* d_out = nullptr;      // its device alias
  size_t off_h = 0, off_c = 0, off_act = 0, off_qa = 0;
  std::vector<cudaGraphExec_t> graphs;   // per row count n
  std::vector<void*> allocs;
  std::recursive_mutex mu;
};
#define DRL_R2_POLICY_LOCK(h) std::lock_guard<std::recursive_mutex> _drl_r2_policy_lock((h)->mu)

namespace {

int check_r2_policy(const drl_r2d2_policy* h) {
  if (!h) { set_error("null r2d2 policy handle"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

// embedding table and conv weight images of the current parameters, on the policy's stream
int refresh_derived(drl_r2d2_policy* h) {
  const R2Layout& pl = h->pl;
  const float* P = h->params;
  DRL_TRY(emb_forward(h->stream, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, h->e1, h->table, h->A));
  return r2_conv_images(h->stream, pl, P, h->img_conv2, h->img_conv3);
}

int enqueue_act(drl_r2d2_policy* h, int n) {
  const R2InLayout l = r2_in_layout(n, h->frame);
  const R2Layout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, l.total, cudaMemcpyHostToDevice, s));
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  const float* h0 = reinterpret_cast<const float*>(h->d_in + l.h0);
  int launches = 0;
  DRL_TRY(r2_conv_forward(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, 1, h->a1, h->a2, h->a3,
                          kR2ConvMode, false, nullptr, &launches));
  DRL_TRY((launch_policy_lstm<kR2L, kR2Splits>(s, h->a3, h->table, pa, h0, P + pl.lstm_w, h->zpart, n)));
  R2HeadArgs a;
  a.zpart = h->zpart;
  a.lstm_b = P + pl.lstm_b;
  a.c0 = reinterpret_cast<const float*>(h->d_in + l.c0);
  a.explore = reinterpret_cast<const int32_t*>(h->d_in + l.explore);
  a.q1_w = P + pl.q1_w; a.q1_b = P + pl.q1_b;
  a.value_w = P + pl.value_w; a.value_b = P + pl.value_b;
  a.mean_w = P + pl.mean_w; a.mean_b = P + pl.mean_b;
  a.q = reinterpret_cast<float*>(h->d_out);
  a.h1 = reinterpret_cast<float*>(h->d_out + h->off_h);
  a.c1 = reinterpret_cast<float*>(h->d_out + h->off_c);
  a.action = reinterpret_cast<int32_t*>(h->d_out + h->off_act);
  a.q_action = reinterpret_cast<float*>(h->d_out + h->off_qa);
  a.n = n;
  a.A = h->A;
  DRL_CUDA_CHECK((launch_k(r2d2_policy_head_kernel, n, kR2G, 0, s, a)));
  return DRL_OK;
}

}  // namespace

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
  if (drl_device_count() <= cfg->device || cfg->device < 0) {
    set_error("CUDA device %d not available (no CPU fallback)", cfg->device);
    return DRL_ERR_CUDA;
  }
  R2PolicyNvtx nv("drl:r2d2_policy_create");
  drl_r2d2_policy* h = new drl_r2d2_policy();
  h->cfg = *cfg;
  h->A = cfg->num_action;
  h->frame = (size_t)Geo::IH * Geo::IW * cfg->channels;
  h->pl.init(h->A, cfg->channels);
  const int MB = cfg->max_batch;
  int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(cfg->device));
    DRL_TRY((set_policy_lstm_attributes<kR2L, kR2Splits>()));
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_ready, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_copied, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreate(&h->ev_start));
    DRL_CUDA_CHECK(cudaEventCreate(&h->ev_stop));
    DRL_TRY(dev_alloc(h, &h->params, (size_t)h->pl.padded_total));
    size_t wb[WeightImages::kCount];
    weight_image_sizes(wb);
    DRL_TRY(dev_alloc(h, &h->img_conv2, wb[1]));
    DRL_TRY(dev_alloc(h, &h->img_conv3, wb[2]));
    DRL_TRY(dev_alloc(h, &h->e1, (size_t)h->A * Geo::EMB));
    DRL_TRY(dev_alloc(h, &h->table, (size_t)h->A * Geo::EMB));
    DRL_TRY(dev_alloc(h, &h->a1, (size_t)MB * 400 * 32));
    DRL_TRY(dev_alloc(h, &h->a2, (size_t)MB * 81 * 64));
    DRL_TRY(dev_alloc(h, &h->a3, (size_t)MB * Geo::FLAT));
    DRL_TRY(dev_alloc(h, &h->zpart, (size_t)kR2Splits * MB * kR2G));
    const size_t in_bytes = r2_in_layout(MB, h->frame).total;
    DRL_TRY(dev_alloc(h, &h->d_in, in_bytes));
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_in, in_bytes, cudaHostAllocDefault));
    memset(h->h_in, 0, in_bytes);
    h->off_h = align_up((size_t)MB * kR2MaxA * 4, 256);
    h->off_c = h->off_h + align_up((size_t)MB * kR2L * 4, 256);
    h->off_act = h->off_c + align_up((size_t)MB * kR2L * 4, 256);
    h->off_qa = h->off_act + align_up((size_t)MB * 4, 256);
    const size_t out_bytes = h->off_qa + align_up((size_t)MB * 4, 256);
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_out, out_bytes, cudaHostAllocMapped));
    memset(h->h_out, 0, out_bytes);
    DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_out, h->h_out, 0));
    h->graphs.assign(MB + 1, nullptr);
    DRL_TRY(refresh_derived(h));   // zero parameters until set_params / sync
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_r2d2_policy_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_r2d2_policy_destroy(drl_r2d2_policy* h) {
  if (!h) return DRL_OK;
  cudaSetDevice(h->cfg.device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto g : h->graphs) if (g) cudaGraphExecDestroy(g);
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_in) cudaFreeHost(h->h_in);
  if (h->h_out) cudaFreeHost(h->h_out);
  for (cudaEvent_t e : {h->ev_ready, h->ev_copied, h->ev_start, h->ev_stop}) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  cudaGetLastError();
  delete h;
  return DRL_OK;
}

int drl_r2d2_policy_param_count(const drl_r2d2_policy* h, int64_t* n) {
  DRL_TRY(check_r2_policy(h));
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->pl.packed_total;
  return DRL_OK;
}

int drl_r2d2_policy_set_params(drl_r2d2_policy* h, const float* host_flat, int64_t n) {
  DRL_TRY(check_r2_policy(h));
  DRL_R2_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("set_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  R2PolicyNvtx nv("drl:r2d2_policy_set_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  DRL_TRY(upload_flat(h->stream, flat.data(), h->pl, h->params, host_flat, 0.0f));
  DRL_TRY(refresh_derived(h));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return DRL_OK;
}

int drl_r2d2_policy_get_params(drl_r2d2_policy* h, float* host_flat, int64_t n) {
  DRL_TRY(check_r2_policy(h));
  DRL_R2_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("get_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  R2PolicyNvtx nv("drl:r2d2_policy_get_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  return download_flat(h->stream, flat.data(), h->pl, h->params, host_flat);
}

int drl_r2d2_policy_sync_from_learner(drl_r2d2_policy* h, drl_r2d2* learner) {
  DRL_TRY(check_r2_policy(h));
  DRL_R2_POLICY_LOCK(h);
  if (!learner) { set_error("null learner handle"); return DRL_ERR_INVALID; }
  R2PolicyNvtx nv("drl:r2d2_policy_sync");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_TRY(r2d2_params_snapshot(learner, h->cfg.device, h->A, h->cfg.channels, h->stream, h->params, h->ev_ready,
                               h->ev_copied));
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  return refresh_derived(h);
}

int drl_r2d2_policy_act(drl_r2d2_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const float* h_in, const float* c_in, const int32_t* explore_action, int32_t* action, float* q,
                        float* q_action, float* h_out, float* c_out) {
  DRL_TRY(check_r2_policy(h));
  DRL_R2_POLICY_LOCK(h);
  if (n < 1 || n > h->cfg.max_batch) { set_error("act: n must be in [1, %d] (got %d)", h->cfg.max_batch, n); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !h_in || !c_in) { set_error("act: null input pointer"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i) {
    if (previous_action[i] < 0 || previous_action[i] >= h->A) {
      set_error("act: previous_action[%d] = %d is outside [0, %d)", i, previous_action[i], h->A);
      return DRL_ERR_INVALID;
    }
    if (explore_action && (explore_action[i] < -1 || explore_action[i] >= h->A)) {
      set_error("act: explore_action[%d] = %d is outside [-1, %d)", i, explore_action[i], h->A);
      return DRL_ERR_INVALID;
    }
  }
  R2PolicyNvtx nv("drl:r2d2_policy_act");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  // the previous call has completed (this entry point is synchronous): the staging block is free
  const R2InLayout l = r2_in_layout(n, h->frame);
  memcpy(h->h_in + l.frames, state, (size_t)n * h->frame);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
  memcpy(h->h_in + l.h0, h_in, (size_t)n * kR2L * 4);
  memcpy(h->h_in + l.c0, c_in, (size_t)n * kR2L * 4);
  if (explore_action) memcpy(h->h_in + l.explore, explore_action, (size_t)n * 4);
  else memset(h->h_in + l.explore, 0xff, (size_t)n * 4);     // -1: greedy
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->stream));
  if (h->cfg.use_cuda_graph) {
    if (!h->graphs[n]) {
      // one eager pass first: the launchers set their kernel attributes outside capture
      DRL_TRY(enqueue_act(h, n));
      DRL_TRY(capture_graph(h->stream, [&] { return enqueue_act(h, n); }, &h->graphs[n]));
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graphs[n], h->stream));
  } else {
    DRL_TRY(enqueue_act(h, n));
  }
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->stream));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->timed = true;
  const int A = h->A;
  if (q) memcpy(q, h->h_out, (size_t)n * A * 4);
  if (h_out) memcpy(h_out, h->h_out + h->off_h, (size_t)n * kR2L * 4);
  if (c_out) memcpy(c_out, h->h_out + h->off_c, (size_t)n * kR2L * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
  if (q_action) memcpy(q_action, h->h_out + h->off_qa, (size_t)n * 4);
  return DRL_OK;
}

int drl_r2d2_policy_last_act_ms(drl_r2d2_policy* h, float* ms) {
  DRL_TRY(check_r2_policy(h));
  DRL_R2_POLICY_LOCK(h);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (!h->timed) { set_error("last_act_ms: no act call has run yet"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

}  // extern "C"
