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
//   conv1 / conv2 / conv3   the Ape-X learner's math-mode-2 kernels and configurations (apex.cu: apex_conv_forward)
//   skinny_splitk_fwd       z = [a3 | table[pa]] [W1_value | W1_mean] (Ape-X, N = 512) or [a3 | table[pa]] W1_actor
//                           (A3C, N = 256) as a skinny split-K FP32-FFMA GEMM (K = 3392, policy_lstm.cuh)
//   apex_policy_head        split-K sum + bias + ReLU, the 256 x 256 layer(s), the output layer(s) and the action rule;
//                           writes q / policy, action and q[action] / policy[action] straight into mapped pinned
//                           memory (no D2H node)
// Both new kernels sum in a fixed order without atomics: eager and graph replays, and repeated calls, are bitwise equal.
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "apex_defs.cuh"
#include "policy_head.cuh"
#include "policy_lstm.cuh"

namespace drl {
namespace {

struct ApexPolicyNvtx {
  explicit ApexPolicyNvtx(const char* name) { nvtxRangePushA(name); }
  ~ApexPolicyNvtx() { nvtxRangePop(); }
};

constexpr int kMaxApexPolicyRows = 64;
constexpr int kApexMaxA = 32;
constexpr int kApexConvMode = 2;   // the learner's default math mode (wgmma 3xTF32 convolutions on weight images)

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

struct drl_apex_policy {
  drl_apex_policy_config cfg{};
  int A = 0;
  ApexLayout pl{};
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_ready = nullptr, ev_copied = nullptr;   // learner -> policy and policy -> learner edges of a sync
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;     // device time of the last act
  bool timed = false;
  float* params = nullptr;       // padded one-network vector (learner layout)
  uint8_t* img_conv2 = nullptr;  // conv2 / conv3 forward weight images (math mode 2)
  uint8_t* img_conv3 = nullptr;
  float* e1 = nullptr;           // [A,256] relu(emb1), scratch of emb_forward
  float* table = nullptr;        // [A,256] action-embedding table (depends on the parameters only)
  float *a1 = nullptr, *a2 = nullptr, *a3 = nullptr;
  float* zpart = nullptr;        // [kApexSplits][max_batch][N]
  uint8_t* d_in = nullptr;       // device input block (apex_in_layout)
  uint8_t* h_in = nullptr;       // pinned staging of the same block
  uint8_t* h_out = nullptr;      // mapped pinned outputs: q / policy [max_batch][A] | action | q[action] / policy[action]
  uint8_t* d_out = nullptr;      // its device alias
  size_t off_act = 0, off_sel = 0;
  std::vector<cudaGraphExec_t> graphs;   // per row count n
  std::vector<void*> allocs;
  std::recursive_mutex mu;
};
#define DRL_APEX_POLICY_LOCK(h) std::lock_guard<std::recursive_mutex> _drl_apex_policy_lock((h)->mu)

namespace {

int check_apex_policy(const drl_apex_policy* h) {
  if (!h) { set_error("null apex policy handle"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

// embedding table and conv weight images of the current parameters, on the policy's stream
int refresh_derived(drl_apex_policy* h) {
  const ApexLayout& pl = h->pl;
  const float* P = h->params;
  DRL_TRY(emb_forward(h->stream, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, h->e1, h->table, h->A));
  return apex_conv_images(h->stream, pl, P, h->img_conv2, h->img_conv3);
}

int enqueue_act(drl_apex_policy* h, int n) {
  const ApexInLayout l = apex_in_layout(n);
  const ApexLayout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, l.total, cudaMemcpyHostToDevice, s));
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  int launches = 0;
  DRL_TRY(apex_conv_forward(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, h->a1, h->a2, h->a3,
                            kApexConvMode, false, nullptr, &launches));
  ApexHeadArgs a;
  a.zpart = h->zpart;
  a.b1v = P + pl.value1_b; a.b1m = P + pl.mean1_b;
  a.w2v = P + pl.value2_w; a.b2v = P + pl.value2_b;
  a.w2m = P + pl.mean2_w; a.b2m = P + pl.mean2_b;
  a.w3v = P + pl.value3_w; a.b3v = P + pl.value3_b;
  a.w3m = P + pl.mean3_w; a.b3m = P + pl.mean3_b;
  a.explore = reinterpret_cast<const int32_t*>(h->d_in + l.sel);
  a.uniform = reinterpret_cast<const double*>(h->d_in + l.sel);
  a.out = reinterpret_cast<float*>(h->d_out);
  a.action = reinterpret_cast<int32_t*>(h->d_out + h->off_act);
  a.out_action = reinterpret_cast<float*>(h->d_out + h->off_sel);
  a.n = n;
  a.A = h->A;
  const int grid = cdiv(n, kHR);
  if (h->cfg.algo == 0) {
    DRL_TRY(launch_head1<0>(s, h->a3, h->table, pa, P + pl.value1_w, P + pl.mean1_w, h->zpart, n));
    DRL_CUDA_CHECK((launch_k(apex_policy_head_kernel<0>, grid, kApexHeadThreads, apex_head_smem<0>(), s, a)));
  } else {
    DRL_TRY(launch_head1<1>(s, h->a3, h->table, pa, P + pl.value1_w, nullptr, h->zpart, n));
    DRL_CUDA_CHECK((launch_k(apex_policy_head_kernel<1>, grid, kApexHeadThreads, apex_head_smem<1>(), s, a)));
  }
  return DRL_OK;
}

// checks common to both act entry points; on success the caller stages `sel` and calls run_act
int check_act(drl_apex_policy* h, int algo, int32_t n, const uint8_t* state, const int32_t* previous_action) {
  if (h->cfg.algo != algo) {
    set_error("act: this policy is %s, use %s", h->cfg.algo ? "A3C" : "Ape-X",
              h->cfg.algo ? "drl_a3c_policy_act" : "drl_apex_policy_act");
    return DRL_ERR_INVALID;
  }
  if (n < 1 || n > h->cfg.max_batch) { set_error("act: n must be in [1, %d] (got %d)", h->cfg.max_batch, n); return DRL_ERR_INVALID; }
  if (!state || !previous_action) { set_error("act: null input pointer"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i) {
    if (previous_action[i] < 0 || previous_action[i] >= h->A) {
      set_error("act: previous_action[%d] = %d is outside [0, %d)", i, previous_action[i], h->A);
      return DRL_ERR_INVALID;
    }
  }
  return DRL_OK;
}

// stages frames and previous actions (the row selectors are already staged), runs the call, copies the outputs out
int run_act(drl_apex_policy* h, int n, const uint8_t* state, const int32_t* previous_action, int32_t* action,
            float* out, float* out_action) {
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  const ApexInLayout l = apex_in_layout(n);
  memcpy(h->h_in + l.frames, state, (size_t)n * Geo::FRAME);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
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
  if (out) memcpy(out, h->h_out, (size_t)n * h->A * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
  if (out_action) memcpy(out_action, h->h_out + h->off_sel, (size_t)n * 4);
  return DRL_OK;
}

}  // namespace

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
  if (drl_device_count() <= cfg->device || cfg->device < 0) {
    set_error("CUDA device %d not available (no CPU fallback)", cfg->device);
    return DRL_ERR_CUDA;
  }
  ApexPolicyNvtx nv("drl:apex_policy_create");
  drl_apex_policy* h = new drl_apex_policy();
  h->cfg = *cfg;
  h->A = cfg->num_action;
  h->pl.init(h->A);
  const int MB = cfg->max_batch;
  int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(cfg->device));
    DRL_TRY(set_apex_policy_kernel_attributes());
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
    DRL_TRY(dev_alloc(h, &h->zpart, (size_t)kApexSplits * MB * (cfg->algo == 0 ? ApexAlgo<0>::N : ApexAlgo<1>::N)));
    const size_t in_bytes = apex_in_layout(MB).total;
    DRL_TRY(dev_alloc(h, &h->d_in, in_bytes));
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_in, in_bytes, cudaHostAllocDefault));
    memset(h->h_in, 0, in_bytes);
    h->off_act = align_up((size_t)MB * kApexMaxA * 4, 256);
    h->off_sel = h->off_act + align_up((size_t)MB * 4, 256);
    const size_t out_bytes = h->off_sel + align_up((size_t)MB * 4, 256);
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
    drl_apex_policy_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_apex_policy_destroy(drl_apex_policy* h) {
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

int drl_apex_policy_param_count(const drl_apex_policy* h, int64_t* n) {
  DRL_TRY(check_apex_policy(h));
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->pl.packed_total;
  return DRL_OK;
}

int drl_apex_policy_set_params(drl_apex_policy* h, const float* host_flat, int64_t n) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("set_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  ApexPolicyNvtx nv("drl:apex_policy_set_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  DRL_TRY(upload_flat(h->stream, flat.data(), h->pl, h->params, host_flat, 0.0f));
  DRL_TRY(refresh_derived(h));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return DRL_OK;
}

int drl_apex_policy_get_params(drl_apex_policy* h, float* host_flat, int64_t n) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("get_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  ApexPolicyNvtx nv("drl:apex_policy_get_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  return download_flat(h->stream, flat.data(), h->pl, h->params, host_flat);
}

int drl_apex_policy_sync_from_learner(drl_apex_policy* h, drl_apex* learner) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  if (!learner) { set_error("null learner handle"); return DRL_ERR_INVALID; }
  ApexPolicyNvtx nv("drl:apex_policy_sync");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_TRY(apex_params_snapshot(learner, h->cfg.device, h->cfg.algo, h->A, h->stream, h->params, h->ev_ready,
                               h->ev_copied));
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  return refresh_derived(h);
}

int drl_apex_policy_act(drl_apex_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const int32_t* explore_action, int32_t* action, float* q, float* q_action) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  DRL_TRY(check_act(h, 0, n, state, previous_action));
  if (explore_action) {
    for (int i = 0; i < n; ++i) {
      if (explore_action[i] < -1 || explore_action[i] >= h->A) {
        set_error("act: explore_action[%d] = %d is outside [-1, %d)", i, explore_action[i], h->A);
        return DRL_ERR_INVALID;
      }
    }
  }
  ApexPolicyNvtx nv("drl:apex_policy_act");
  // the previous call has completed (this entry point is synchronous): the staging block is free
  uint8_t* sel = h->h_in + apex_in_layout(n).sel;
  if (explore_action) memcpy(sel, explore_action, (size_t)n * 4);
  else memset(sel, 0xff, (size_t)n * 4);      // -1: greedy
  return run_act(h, n, state, previous_action, action, q, q_action);
}

int drl_a3c_policy_act(drl_a3c_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                       const double* uniform, int32_t* action, float* policy, float* prob_action) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  DRL_TRY(check_act(h, 1, n, state, previous_action));
  if (!uniform) { set_error("act: null input pointer (uniform: one draw in [0, 1) per row)"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i) {
    if (!(uniform[i] >= 0.0 && uniform[i] < 1.0)) {
      set_error("act: uniform[%d] = %g is outside [0, 1)", i, uniform[i]);
      return DRL_ERR_INVALID;
    }
  }
  ApexPolicyNvtx nv("drl:a3c_policy_act");
  memcpy(h->h_in + apex_in_layout(n).sel, uniform, (size_t)n * 8);
  return run_act(h, n, state, previous_action, action, policy, prob_action);
}

int drl_apex_policy_last_act_ms(drl_apex_policy* h, float* ms) {
  DRL_TRY(check_apex_policy(h));
  DRL_APEX_POLICY_LOCK(h);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (!h->timed) { set_error("last_act_ms: no act call has run yet"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

}  // extern "C"
