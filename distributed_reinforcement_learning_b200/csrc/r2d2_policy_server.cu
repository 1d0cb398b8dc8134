// r2d2_policy_server.cu -- the R2D2 policy server behind drl_r2d2_policy_server_* (include/drl_b200.h; DESIGN.md
// section 17).  One R2D2 engine (r2d2_policy.cu) serves environments that step in other processes.  Each environment's
// h, c, previous action and step live in a device state table and its unfinished sequence in a device staging indexed
// by environment, in the R2D2 queue's field order (R2QueueField); the processes exchange frames and actions with the
// server through the same exchange block as the IMPALA server (server_core.cuh), with DRL_R2D2_SERVER_* records.
//
// One serve of n rows = one upload of the call's word block (env ids, completed-row list, explore actions) + on the
// engine's stream:
//   r2d2_server_gather_kernel    report -> the engine's device input rows (frame; h, c, previous action from the
//                                table, or 0 on reset; the explore action the host checked); the previous step's
//                                reward and done -> staging at (t - 1) mod S
//   queue_commit_rows_kernel     the staged sequences that step S-1 completed -> their reserved queue positions
//                                (server_core.cu)
//   the engine's act kernels     (r2d2_policy_enqueue_forward: conv stack, policy_lstm_fwd, r2d2_policy_head), outputs
//                                into device memory
//   r2d2_server_scatter_kernel   step t of each row into the staging (frame, previous action, action; at t = 0 h0 and
//                                c0); h, c, previous action, t into the table; action and q_action into the reply
// The graph pair per n, the reservation and the commit events are the server core's.
//
// The explore action comes from another process and the head indexes q with it, so the host reads it once from the
// block, checks it against [-1, A) and stages the checked value in the word block; the kernels never read it from the
// report.  A bad value fails the serve before anything is reserved or launched.
#include "r2d2_defs.cuh"
#include "server_core.cuh"

namespace drl {
namespace {

constexpr int kThreads = kServerThreads;

static_assert(DRL_R2D2_SERVER_REPORT_BYTES == DRL_SERVER_REPORT_BYTES &&
                  DRL_R2D2_SERVER_REPLY_BYTES == DRL_SERVER_REPLY_BYTES,
              "one exchange block size for both servers");
static_assert(DRL_R2D2_SERVER_REPORT_FRAME == 0 && DRL_R2D2_SERVER_REPORT_EXPLORE >= Geo::IH * Geo::IW * 4,
              "the report keeps 84x84x4 bytes for the frame at either C");
static_assert(DRL_R2D2_SERVER_REPORT_REWARD % 16 == 0 && DRL_R2D2_SERVER_REPORT_DONE % 16 == 0 &&
                  DRL_R2D2_SERVER_REPORT_RESET % 16 == 0 && DRL_R2D2_SERVER_REPLY_Q_ACTION % 16 == 0,
              "16-byte aligned fields");

struct R2Table {
  float* h;          // [num_envs][64]
  float* c;          // [num_envs][64]
  int32_t* pa;       // [num_envs]
  int32_t* t;        // [num_envs]: the step the next act records, -1 before the first
};

// ---- r2d2_server_gather_kernel ----------------------------------------------------------------------------------
struct R2GatherArgs {
  const uint8_t* reports;    // mapped exchange block
  const int32_t* env;        // [n]
  const int32_t* explore;    // [n]: checked by the host
  R2Table tab;
  R2PolicyInRows in;
  float* st_reward;          // staging [num_envs][S]
  uint8_t* st_done;          // [num_envs][S]
  int S;
};

// kFrame16: 16-byte vectors of the queue's frame (441 at C = 1, 1764 at C = 4)
template <int kFrame16>
__global__ void __launch_bounds__(kThreads) r2d2_server_gather_kernel(const R2GatherArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  const uint8_t* rep = a.reports + (size_t)e * DRL_R2D2_SERVER_REPORT_BYTES;
  // every load of the frame issued before the first store: each is a round trip over PCIe
  const uint4* f = reinterpret_cast<const uint4*>(rep + DRL_R2D2_SERVER_REPORT_FRAME);
  uint4* fd = reinterpret_cast<uint4*>(a.in.frames) + (size_t)row * kFrame16;
  constexpr int kPer = (kFrame16 + kThreads - 1) / kThreads;
  uint4 v[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kFrame16) v[k] = f[tid + k * kThreads];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kFrame16) fd[tid + k * kThreads] = v[k];
  // one 16-byte load per scalar field of the report
  const bool reset = reinterpret_cast<const uint4*>(rep + DRL_R2D2_SERVER_REPORT_RESET)->x & 0xffu;
  if (tid < kR2L / 4) {
    const float4 x = reset ? zero4() : reinterpret_cast<const float4*>(a.tab.h + (size_t)e * kR2L)[tid];
    reinterpret_cast<float4*>(a.in.h0 + (size_t)row * kR2L)[tid] = x;
  } else if (tid < kR2L / 2) {
    const int i = tid - kR2L / 4;
    const float4 x = reset ? zero4() : reinterpret_cast<const float4*>(a.tab.c + (size_t)e * kR2L)[i];
    reinterpret_cast<float4*>(a.in.c0 + (size_t)row * kR2L)[i] = x;
  } else if (tid == kR2L / 2) {
    a.in.pa[row] = reset ? 0 : a.tab.pa[e];
  } else if (tid == kR2L / 2 + 1) {
    a.in.explore[row] = a.explore[row];
  } else if (tid == kR2L / 2 + 2) {
    const int t = a.tab.t[e];
    if (t >= 0) {   // the reward and done of the previous step (t - 1, or S - 1 of the sequence step t = 0 follows)
      const size_t prev = (size_t)e * a.S + (t + a.S - 1) % a.S;
      const uint4 r = *reinterpret_cast<const uint4*>(rep + DRL_R2D2_SERVER_REPORT_REWARD);
      const uint4 d = *reinterpret_cast<const uint4*>(rep + DRL_R2D2_SERVER_REPORT_DONE);
      a.st_reward[prev] = __uint_as_float(r.x);
      a.st_done[prev] = (uint8_t)(d.x & 0xffu);
    }
  }
}

// ---- r2d2_server_scatter_kernel ---------------------------------------------------------------------------------
struct R2ScatterArgs {
  const int32_t* env;        // [n]
  R2PolicyInRows in;         // what the act read
  R2PolicyOutRows out;       // what it computed (device)
  R2Table tab;
  uint8_t* st_frames;        // staging [num_envs][S][frame]
  int32_t* st_pa;            // [num_envs][S]
  int32_t* st_action;        // [num_envs][S]
  float* st_h;               // [num_envs][64]: step 0 only
  float* st_c;               // [num_envs][64]
  uint8_t* replies;          // mapped reply records
  int S;
};

template <int kFrame16>
__global__ void __launch_bounds__(kThreads) r2d2_server_scatter_kernel(const R2ScatterArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  // every thread reads the step before the barrier below; the table's step is written only after it
  const int t = max(a.tab.t[e], 0);
  const size_t dst = (size_t)e * a.S + t;
  if (tid < kR2L / 4) {
    if (t == 0)
      reinterpret_cast<float4*>(a.st_h + (size_t)e * kR2L)[tid] =
          reinterpret_cast<const float4*>(a.in.h0 + (size_t)row * kR2L)[tid];
    reinterpret_cast<float4*>(a.tab.h + (size_t)e * kR2L)[tid] =
        reinterpret_cast<const float4*>(a.out.h1 + (size_t)row * kR2L)[tid];
  } else if (tid < kR2L / 2) {
    const int i = tid - kR2L / 4;
    if (t == 0)
      reinterpret_cast<float4*>(a.st_c + (size_t)e * kR2L)[i] =
          reinterpret_cast<const float4*>(a.in.c0 + (size_t)row * kR2L)[i];
    reinterpret_cast<float4*>(a.tab.c + (size_t)e * kR2L)[i] =
        reinterpret_cast<const float4*>(a.out.c1 + (size_t)row * kR2L)[i];
  } else if (tid == kR2L / 2) {
    const int32_t act = a.out.action[row];
    a.st_pa[dst] = a.in.pa[row];
    a.st_action[dst] = act;
    a.tab.pa[e] = act;
    uint8_t* rep = a.replies + (size_t)e * DRL_R2D2_SERVER_REPLY_BYTES;
    *reinterpret_cast<int32_t*>(rep + DRL_R2D2_SERVER_REPLY_ACTION) = act;
    *reinterpret_cast<float*>(rep + DRL_R2D2_SERVER_REPLY_Q_ACTION) = a.out.q_action[row];
  }
  const uint4* f = reinterpret_cast<const uint4*>(a.in.frames) + (size_t)row * kFrame16;
  uint4* fd = reinterpret_cast<uint4*>(a.st_frames) + dst * kFrame16;
  constexpr int kPer = (kFrame16 + kThreads - 1) / kThreads;
  uint4 v[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kFrame16) v[k] = f[tid + k * kThreads];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kFrame16) fd[tid + k * kThreads] = v[k];
  __syncthreads();
  if (tid == 0) a.tab.t[e] = (t + 1) % a.S;
}

constexpr int kFrame16C1 = Geo::IH * Geo::IW * 1 / 16;
constexpr int kFrame16C4 = Geo::IH * Geo::IW * 4 / 16;

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_r2d2_policy_server : ServerCore {
  drl_r2d2_policy* policy = nullptr;
  int C = 1;
  R2Table tab{};
  float* out_q = nullptr;             // the act's outputs [max_batch][A] / [max_batch][64] / [max_batch]
  float *out_h = nullptr, *out_c = nullptr;
  int32_t* out_action = nullptr;
  float* out_qa = nullptr;
};

namespace {

// the explore action of each row, read once from its report, checked, and staged in the word block
int stage_explore(ServerCore* s, int n, const int32_t* env_ids) {
  const int A = s->engine->A;
  int32_t* w = s->h_words + s->words.extra_words();
  for (int r = 0; r < n; ++r) {
    const int e = env_ids[r];
    const int32_t x = *reinterpret_cast<const volatile int32_t*>(
        s->host_block + (size_t)e * DRL_R2D2_SERVER_REPORT_BYTES + DRL_R2D2_SERVER_REPORT_EXPLORE);
    if (x < -1 || x >= A) {
      set_error("%s serve: environment %d reports explore action %d, outside [-1, %d)", s->name, e, x, A);
      return DRL_ERR_INVALID;
    }
    w[r] = x;
  }
  return DRL_OK;
}

// the kernels of the queue's frame size
int launch_gather(drl_r2d2_policy_server* s, int n, const R2GatherArgs& g) {
  auto k = s->C == 1 ? r2d2_server_gather_kernel<kFrame16C1> : r2d2_server_gather_kernel<kFrame16C4>;
  DRL_CUDA_CHECK((launch_k(k, n, kThreads, 0, s->engine->stream, g)));
  return DRL_OK;
}

int launch_scatter(drl_r2d2_policy_server* s, int n, const R2ScatterArgs& a) {
  auto k = s->C == 1 ? r2d2_server_scatter_kernel<kFrame16C1> : r2d2_server_scatter_kernel<kFrame16C4>;
  DRL_CUDA_CHECK((launch_k(k, n, kThreads, 0, s->engine->stream, a)));
  return DRL_OK;
}

// the serve of n rows; `commit`: with queue_commit_rows_kernel (some row completes a sequence)
int enqueue_serve(ServerCore* core, int n, bool commit) {
  drl_r2d2_policy_server* s = static_cast<drl_r2d2_policy_server*>(core);
  DRL_TRY(server_upload_words(s));
  const R2PolicyInRows in = r2d2_policy_input_rows(s->policy, n);
  const int32_t* env = s->d_words + s->words.env();
  R2GatherArgs g;
  g.reports = s->d_block;
  g.env = env;
  g.explore = s->d_words + s->words.extra_words();
  g.tab = s->tab;
  g.in = in;
  g.st_reward = reinterpret_cast<float*>(s->st[kR2QReward]);
  g.st_done = s->st[kR2QDone];
  g.S = s->T;
  R2ScatterArgs a;
  a.env = env;
  a.in = in;
  a.out = R2PolicyOutRows{s->out_q, s->out_h, s->out_c, s->out_action, s->out_qa};
  a.tab = s->tab;
  a.st_frames = s->st[kR2QFrames];
  a.st_pa = reinterpret_cast<int32_t*>(s->st[kR2QPa]);
  a.st_action = reinterpret_cast<int32_t*>(s->st[kR2QAction]);
  a.st_h = reinterpret_cast<float*>(s->st[kR2QH]);
  a.st_c = reinterpret_cast<float*>(s->st[kR2QC]);
  a.replies = s->d_block + (size_t)s->num_envs * DRL_R2D2_SERVER_REPORT_BYTES;
  a.S = s->T;
  DRL_TRY(launch_gather(s, n, g));
  if (commit) DRL_TRY(server_enqueue_commit(s, n));
  DRL_TRY(r2d2_policy_enqueue_forward(s->policy, n, a.out));
  DRL_TRY(launch_scatter(s, n, a));
  return DRL_OK;
}

int server_init(drl_r2d2_policy_server* s, void* exchange) {
  DRL_TRY(server_core_init(s, exchange));
  PolicyCore* h = s->engine;
  const size_t E = s->num_envs, MB = h->max_batch;
  DRL_TRY(dev_alloc(s, &s->tab.h, E * kR2L));
  DRL_TRY(dev_alloc(s, &s->tab.c, E * kR2L));
  DRL_TRY(dev_alloc(s, &s->tab.pa, E));
  DRL_TRY(dev_alloc(s, &s->tab.t, E, 0xff));   // -1: no step yet
  DRL_TRY(dev_alloc(s, &s->out_q, MB * h->A));
  DRL_TRY(dev_alloc(s, &s->out_h, MB * kR2L));
  DRL_TRY(dev_alloc(s, &s->out_c, MB * kR2L));
  DRL_TRY(dev_alloc(s, &s->out_action, MB));
  DRL_TRY(dev_alloc(s, &s->out_qa, MB));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_r2d2_policy_server_create(drl_r2d2_policy* p, drl_r2d2_queue* q, int32_t num_envs, void* exchange,
                                  int64_t exchange_size, drl_r2d2_policy_server** out) {
  constexpr const char* kName = "r2d2 policy server";
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  if (!p) { set_error("null r2d2 policy handle"); return DRL_ERR_INVALID; }
  if (!q) { set_error("null r2d2 queue handle"); return DRL_ERR_INVALID; }
  DRL_TRY(server_check_block(kName, num_envs, DRL_SERVER_REPORT_BYTES, exchange, exchange_size));
  PolicyCore* h = r2d2_policy_core_of(p);
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (q->device != h->device) {
    set_error("%s: the queue is on device %d, the policy on device %d", kName, q->device, h->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != h->A) { set_error("%s: the queue has num_action %d, the policy %d", kName, q->A, h->A); return DRL_ERR_INVALID; }
  const int C = r2d2_policy_channels(p);
  if (q->C != C) {
    set_error("%s: the queue stores 84x84x%d frames, the policy takes 84x84x%d", kName, q->C, C);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:r2d2_policy_server_create");
  drl_r2d2_policy_server* s = new drl_r2d2_policy_server();
  s->name = kName;
  s->serve_range = "drl:r2d2_policy_server_serve";
  s->policy = p;
  s->engine = h;
  s->q = q;
  s->num_envs = num_envs;
  s->report_bytes = DRL_SERVER_REPORT_BYTES;
  s->T = q->S;
  s->C = C;
  s->enqueue_serve = enqueue_serve;
  s->stage_rows = stage_explore;
  s->extra_words = 1;
  int rc = server_check_queue_rows(s, "sequences");
  if (rc == DRL_OK) rc = server_init(s, exchange);
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    server_core_release(s);
    delete s;
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = s;
  return DRL_OK;
}

int drl_r2d2_policy_server_destroy(drl_r2d2_policy_server* s) { return server_destroy(s); }

int drl_r2d2_policy_server_serve(drl_r2d2_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms) {
  if (!s) { set_error("null r2d2 policy server handle"); return DRL_ERR_INVALID; }
  return server_serve(s, n, env_ids, timeout_ms);
}

}  // extern "C"
