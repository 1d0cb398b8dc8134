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
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "kernels.h"
#include "policy_head.cuh"
#include "policy_lstm.cuh"

namespace drl {
namespace {

struct PolicyNvtx {
  explicit PolicyNvtx(const char* name) { nvtxRangePushA(name); }
  ~PolicyNvtx() { nvtxRangePop(); }
};

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
  return DRL_OK;
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_policy {
  drl_policy_config cfg{};
  int A = 0;
  ParamLayout pl{};
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_ready = nullptr, ev_copied = nullptr;   // learner -> policy and policy -> learner edges of a sync
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;     // device time of the last act
  bool timed = false;
  float* params = nullptr;       // padded flat vector (learner layout)
  uint8_t* img_conv2 = nullptr;  // conv2 / conv3 forward weight images (16-bit split, gemm_umma16.cuh)
  uint8_t* img_conv3 = nullptr;
  float* e1 = nullptr;           // [A,256] relu(emb1), scratch of emb_forward
  float* table = nullptr;        // [A,256] action-embedding table (depends on the parameters only)
  float *a1 = nullptr, *a2 = nullptr, *a3 = nullptr;
  float* zpart = nullptr;        // [kLSplits][max_batch][1024]
  uint8_t* d_in = nullptr;       // device input block (in_layout)
  uint8_t* h_in = nullptr;       // pinned staging of the same block
  uint8_t* h_out = nullptr;      // mapped pinned outputs: policy [max_batch][A] | h1 | c1 [max_batch][256] | action
  uint8_t* d_out = nullptr;      // its device alias
  size_t off_h = 0, off_c = 0, off_act = 0;
  std::vector<cudaGraphExec_t> graphs;   // per row count n
  std::vector<void*> allocs;
  std::recursive_mutex mu;
};
#define DRL_POLICY_LOCK(h) std::lock_guard<std::recursive_mutex> _drl_policy_lock((h)->mu)

namespace {

int check_policy(const drl_policy* h) {
  if (!h) { set_error("null policy handle"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

// embedding table and conv weight images of the current parameters, on the policy's stream
int refresh_derived(drl_policy* h) {
  const ParamLayout& pl = h->pl;
  const float* P = h->params;
  DRL_TRY(emb_forward(h->stream, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, h->e1, h->table, h->A));
  return conv_images16(h->stream, pl, P, h->img_conv2, h->img_conv3);
}

int enqueue_act(drl_policy* h, int n) {
  const InLayout l = in_layout(n);
  const ParamLayout& pl = h->pl;
  const float* P = h->params;
  cudaStream_t s = h->stream;
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->d_in, h->h_in, l.total, cudaMemcpyHostToDevice, s));
  const int32_t* pa = reinterpret_cast<const int32_t*>(h->d_in + l.pa);
  const float* h0 = reinterpret_cast<const float*>(h->d_in + l.h0);
  DRL_TRY(conv_forward16(s, pl, P, h->img_conv2, h->img_conv3, h->d_in + l.frames, n, h->a1, h->a2, h->a3));
  DRL_TRY((launch_policy_lstm<Geo::L, kLSplits>(s, h->a3, h->table, pa, h0, P + pl.lstm_w, h->zpart, n)));
  HeadArgs a;
  a.zpart = h->zpart;
  a.lstm_b = P + pl.lstm_b;
  a.c0 = reinterpret_cast<const float*>(h->d_in + l.c0);
  a.uniform = reinterpret_cast<const double*>(h->d_in + l.u);
  a.w1 = P + pl.actor1_w; a.b1 = P + pl.actor1_b;
  a.w2 = P + pl.actor2_w; a.b2 = P + pl.actor2_b;
  a.w3 = P + pl.actor3_w; a.b3 = P + pl.actor3_b;
  a.policy = reinterpret_cast<float*>(h->d_out);
  a.h1 = reinterpret_cast<float*>(h->d_out + h->off_h);
  a.c1 = reinterpret_cast<float*>(h->d_out + h->off_c);
  a.action = reinterpret_cast<int32_t*>(h->d_out + h->off_act);
  a.n = n;
  a.A = h->A;
  DRL_CUDA_CHECK((launch_k(policy_head_fused_kernel, cdiv(n, kHR), kHThreads, kHeadSmem, s, a)));
  return DRL_OK;
}

}  // namespace

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
  if (drl_device_count() <= cfg->device || cfg->device < 0) {
    set_error("CUDA device %d not available (no CPU fallback)", cfg->device);
    return DRL_ERR_CUDA;
  }
  PolicyNvtx nv("drl:policy_create");
  drl_policy* h = new drl_policy();
  h->cfg = *cfg;
  h->A = cfg->num_action;
  h->pl.init(h->A);
  const int MB = cfg->max_batch;
  int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(cfg->device));
    DRL_TRY(set_policy_kernel_attributes());
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
    DRL_TRY(dev_alloc(h, &h->zpart, (size_t)kLSplits * MB * Geo::G4));
    const size_t in_bytes = in_layout(MB).total;
    DRL_TRY(dev_alloc(h, &h->d_in, in_bytes));
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_in, in_bytes, cudaHostAllocDefault));
    memset(h->h_in, 0, in_bytes);
    h->off_h = align_up((size_t)MB * kMaxA * 4, 256);
    h->off_c = h->off_h + align_up((size_t)MB * Geo::L * 4, 256);
    h->off_act = h->off_c + align_up((size_t)MB * Geo::L * 4, 256);
    const size_t out_bytes = h->off_act + align_up((size_t)MB * 4, 256);
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
    drl_policy_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_policy_destroy(drl_policy* h) {
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

int drl_policy_param_count(const drl_policy* h, int64_t* n) {
  DRL_TRY(check_policy(h));
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->pl.packed_total;
  return DRL_OK;
}

int drl_policy_set_params(drl_policy* h, const float* host_flat, int64_t n) {
  DRL_TRY(check_policy(h));
  DRL_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("set_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  PolicyNvtx nv("drl:policy_set_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  DRL_TRY(upload_flat(h->stream, flat.data(), h->pl, h->params, host_flat, 0.0f));
  DRL_TRY(refresh_derived(h));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return DRL_OK;
}

int drl_policy_get_params(drl_policy* h, float* host_flat, int64_t n) {
  DRL_TRY(check_policy(h));
  DRL_POLICY_LOCK(h);
  if (!host_flat || n != h->pl.packed_total) {
    set_error("get_params: expected %lld floats, got %lld", (long long)h->pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  PolicyNvtx nv("drl:policy_get_params");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  std::vector<float> flat((size_t)h->pl.padded_total);
  return download_flat(h->stream, flat.data(), h->pl, h->params, host_flat);
}

int drl_policy_sync_from_learner(drl_policy* h, drl_learner* learner) {
  DRL_TRY(check_policy(h));
  DRL_POLICY_LOCK(h);
  if (!learner) { set_error("null learner handle"); return DRL_ERR_INVALID; }
  PolicyNvtx nv("drl:policy_sync");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_TRY(learner_params_snapshot(learner, h->cfg.device, h->A, h->stream, h->params, h->ev_ready, h->ev_copied));
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  return refresh_derived(h);
}

int drl_policy_act(drl_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
                   const float* c_in, const double* uniform, int32_t* action, float* policy, float* h_out,
                   float* c_out) {
  DRL_TRY(check_policy(h));
  DRL_POLICY_LOCK(h);
  if (n < 1 || n > h->cfg.max_batch) { set_error("act: n must be in [1, %d] (got %d)", h->cfg.max_batch, n); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !h_in || !c_in) { set_error("act: null input pointer"); return DRL_ERR_INVALID; }
  if (action && !uniform) { set_error("act: `action` needs `uniform` (one draw in [0, 1) per row)"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i) {
    if (previous_action[i] < 0 || previous_action[i] >= h->A) {
      set_error("act: previous_action[%d] = %d is outside [0, %d)", i, previous_action[i], h->A);
      return DRL_ERR_INVALID;
    }
  }
  PolicyNvtx nv("drl:policy_act");
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  // the previous call has completed (this entry point is synchronous): the staging block is free
  const InLayout l = in_layout(n);
  memcpy(h->h_in + l.frames, state, (size_t)n * Geo::FRAME);
  memcpy(h->h_in + l.pa, previous_action, (size_t)n * 4);
  memcpy(h->h_in + l.h0, h_in, (size_t)n * Geo::L * 4);
  memcpy(h->h_in + l.c0, c_in, (size_t)n * Geo::L * 4);
  if (uniform) memcpy(h->h_in + l.u, uniform, (size_t)n * 8);
  else memset(h->h_in + l.u, 0, (size_t)n * 8);
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->stream));
  if (h->cfg.use_cuda_graph) {
    if (!h->graphs[n]) {
      // one eager pass first: the launchers set their kernel attributes and build their tensor maps outside capture
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
  if (policy) memcpy(policy, h->h_out, (size_t)n * A * 4);
  if (h_out) memcpy(h_out, h->h_out + h->off_h, (size_t)n * Geo::L * 4);
  if (c_out) memcpy(c_out, h->h_out + h->off_c, (size_t)n * Geo::L * 4);
  if (action) memcpy(action, h->h_out + h->off_act, (size_t)n * 4);
  return DRL_OK;
}

int drl_policy_last_act_ms(drl_policy* h, float* ms) {
  DRL_TRY(check_policy(h));
  DRL_POLICY_LOCK(h);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (!h->timed) { set_error("last_act_ms: no act call has run yet"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(h->cfg.device));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

}  // extern "C"
