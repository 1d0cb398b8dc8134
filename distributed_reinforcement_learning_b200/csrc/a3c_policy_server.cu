// a3c_policy_server.cu -- the A3C policy server behind drl_a3c_policy_server_* (include/drl_b200.h; DESIGN.md section
// 18).  One A3C engine (apex_policy.cu, algo 1) serves environments that step in other processes.  Each environment's
// previous action and step live in a device state table and its unfinished unroll in a device staging indexed by
// environment, in the A3C queue's record layout (ApexQueueField: frames [2T] = state rows then next_state rows,
// pa2 [2T] = previous actions then actions, reward [T], done [T]); the processes exchange frames and actions with the
// server through an exchange block (server_core.cuh) of DRL_A3C_SERVER_* records.
//
// One serve of n rows = one upload of the call's word block (env ids, completed-row list) + on the engine's stream:
//   a3c_server_gather_kernel    report -> the engine's device input rows (frame, uniform; the previous action from the
//                               table, or 0 on reset); the previous step's reward, done and next_state -> staging at
//                               (t - 1) mod T.  That next_state is this report's frame, or its next_state field when
//                               reset is set (the episode ended: the frame to act on is the new episode's first)
//   queue_commit_rows_kernel    the staged unrolls that step T-1 completed -> their reserved queue positions
//                               (server_core.cu)
//   the engine's act kernels    (apex_policy_enqueue_forward: conv stack, skinny_splitk_fwd,
//                               apex_policy_head_kernel<1>), outputs into device memory
//   a3c_server_scatter_kernel   state row t <- the engine's input frame; pa2[t] <- the previous action, pa2[T + t] <-
//                               the action; the table's previous action and t; action and policy[action] into the reply
// Ordering: a record's last next_state row (T - 1), reward and done are written by the gather of the serve whose
// commit copies the record, so they precede the commit; the state row 0 and pa2[0] / pa2[T] of the next unroll
// overwrite the same staging, so the scatter writes them, after the commit.  The graph pair per n, the reservation and
// the commit events are the server core's.
//
// The uniform is read on the device only, as in the IMPALA server: sample_choice clamps the action to [0, A) for any
// value, so nothing the other process writes can index out of bounds.
#include "server_core.cuh"

namespace drl {
namespace {

constexpr int kThreads = kServerThreads;
constexpr int kF16 = Geo::FRAME / 16;                         // 16-byte vectors of one frame
constexpr int kPer = (kF16 + kThreads - 1) / kThreads;

static_assert(DRL_A3C_SERVER_REPORT_FRAME == 0 && DRL_A3C_SERVER_REPORT_NEXT_STATE == Geo::FRAME &&
                  DRL_A3C_SERVER_REPORT_UNIFORM >= 2 * Geo::FRAME, "report layout");
static_assert(DRL_A3C_SERVER_REPORT_UNIFORM % 16 == 0 && DRL_A3C_SERVER_REPORT_REWARD % 16 == 0 &&
                  DRL_A3C_SERVER_REPORT_DONE % 16 == 0 && DRL_A3C_SERVER_REPORT_RESET % 16 == 0 &&
                  DRL_A3C_SERVER_REPORT_BYTES % 16 == 0 && DRL_A3C_SERVER_REPLY_MAX_PROB % 16 == 0,
              "16-byte aligned fields");
static_assert(DRL_A3C_SERVER_REPLY_BYTES == DRL_SERVER_REPLY_BYTES, "the server core's reply stride");

struct A3CTable {
  int32_t* pa;       // [num_envs]
  int32_t* t;        // [num_envs]: the step the next act records, -1 before the first
};

// ---- a3c_server_gather_kernel -----------------------------------------------------------------------------------
struct A3CGatherArgs {
  const uint8_t* reports;    // mapped exchange block
  const int32_t* env;        // [n]
  A3CTable tab;
  ApexPolicyInRows in;
  uint8_t* st_frames;        // staging [num_envs][2T][frame]
  float* st_reward;          // [num_envs][T]
  uint8_t* st_done;          // [num_envs][T]
  int T;
};

__global__ void __launch_bounds__(kThreads) a3c_server_gather_kernel(const A3CGatherArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  const uint8_t* rep = a.reports + (size_t)e * DRL_A3C_SERVER_REPORT_BYTES;
  const int t = a.tab.t[e];
  // one 16-byte load per scalar field of the report
  const bool reset = reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_RESET)->x & 0xffu;
  // the previous step's next_state: the frame to act on, or after an episode end the report's next_state
  const bool prev = t >= 0, from_next = prev && reset;
  // every load of the frames issued before the first store: each is a round trip over PCIe
  const uint4* f = reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_FRAME);
  const uint4* g = reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_NEXT_STATE);
  uint4 v[kPer], w[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kF16) v[k] = f[tid + k * kThreads];
  if (from_next) {
#pragma unroll
    for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kF16) w[k] = g[tid + k * kThreads];
  }
  uint4* fd = reinterpret_cast<uint4*>(a.in.frames) + (size_t)row * kF16;
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kF16) fd[tid + k * kThreads] = v[k];
  if (prev) {   // next_state row (t - 1) mod T: row T - 1 of the unroll this serve's commit copies when t = 0
    uint4* nd = reinterpret_cast<uint4*>(a.st_frames) + ((size_t)e * 2 * a.T + a.T + (t + a.T - 1) % a.T) * kF16;
#pragma unroll
    for (int k = 0; k < kPer; ++k)
      if (tid + k * kThreads < kF16) nd[tid + k * kThreads] = from_next ? w[k] : v[k];
  }
  if (tid == 0) {
    a.in.pa[row] = reset ? 0 : a.tab.pa[e];
  } else if (tid == 1) {
    const uint4 u = *reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_UNIFORM);
    a.in.uniform[row] = __hiloint2double((int)u.y, (int)u.x);
  } else if (tid == 2 && prev) {   // the reward and done of the previous step
    const size_t p = (size_t)e * a.T + (t + a.T - 1) % a.T;
    const uint4 r = *reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_REWARD);
    const uint4 d = *reinterpret_cast<const uint4*>(rep + DRL_A3C_SERVER_REPORT_DONE);
    a.st_reward[p] = __uint_as_float(r.x);
    a.st_done[p] = (uint8_t)(d.x & 0xffu);
  }
}

// ---- a3c_server_scatter_kernel ----------------------------------------------------------------------------------
struct A3CScatterArgs {
  const int32_t* env;        // [n]
  ApexPolicyInRows in;       // what the act read
  ApexPolicyOutRows out;     // what it computed (device)
  A3CTable tab;
  uint8_t* st_frames;        // staging [num_envs][2T][frame]
  int32_t* st_pa2;           // [num_envs][2T]
  uint8_t* replies;          // mapped reply records
  int T;
};

__global__ void __launch_bounds__(kThreads) a3c_server_scatter_kernel(const A3CScatterArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  // every thread reads the step before the barrier below; the table's step is written only after it
  const int t = max(a.tab.t[e], 0);
  if (tid == 0) {
    const int32_t act = a.out.action[row];
    int32_t* pa2 = a.st_pa2 + (size_t)e * 2 * a.T;
    pa2[t] = a.in.pa[row];
    pa2[a.T + t] = act;
    a.tab.pa[e] = act;
    uint8_t* rep = a.replies + (size_t)e * DRL_A3C_SERVER_REPLY_BYTES;
    *reinterpret_cast<int32_t*>(rep + DRL_A3C_SERVER_REPLY_ACTION) = act;
    *reinterpret_cast<float*>(rep + DRL_A3C_SERVER_REPLY_MAX_PROB) = a.out.out_action[row];
  }
  const uint4* f = reinterpret_cast<const uint4*>(a.in.frames) + (size_t)row * kF16;
  uint4* fd = reinterpret_cast<uint4*>(a.st_frames) + ((size_t)e * 2 * a.T + t) * kF16;
  uint4 v[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kF16) v[k] = f[tid + k * kThreads];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < kF16) fd[tid + k * kThreads] = v[k];
  __syncthreads();
  if (tid == 0) a.tab.t[e] = (t + 1) % a.T;
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_a3c_policy_server : ServerCore {
  drl_apex_policy* policy = nullptr;
  A3CTable tab{};
  float* out_policy = nullptr;        // the act's outputs [max_batch][A] / [max_batch] / [max_batch]
  int32_t* out_action = nullptr;
  float* out_prob = nullptr;
};

namespace {

// the serve of n rows; `commit`: with queue_commit_rows_kernel (some row completes an unroll)
int enqueue_serve(ServerCore* core, int n, bool commit) {
  drl_a3c_policy_server* s = static_cast<drl_a3c_policy_server*>(core);
  cudaStream_t st = s->engine->stream;
  DRL_TRY(server_upload_words(s));
  const ApexPolicyInRows in = apex_policy_input_rows(s->policy, n);
  const int32_t* env = s->d_words + s->words.env();
  A3CGatherArgs g;
  g.reports = s->d_block;
  g.env = env;
  g.tab = s->tab;
  g.in = in;
  g.st_frames = s->st[kApexQFrames];
  g.st_reward = reinterpret_cast<float*>(s->st[kApexQReward]);
  g.st_done = s->st[kApexQDone];
  g.T = s->T;
  DRL_CUDA_CHECK((launch_k(a3c_server_gather_kernel, n, kThreads, 0, st, g)));
  if (commit) DRL_TRY(server_enqueue_commit(s, n));
  const ApexPolicyOutRows out{s->out_policy, s->out_action, s->out_prob};
  DRL_TRY(apex_policy_enqueue_forward(s->policy, n, out));
  A3CScatterArgs a;
  a.env = env;
  a.in = in;
  a.out = out;
  a.tab = s->tab;
  a.st_frames = s->st[kApexQFrames];
  a.st_pa2 = reinterpret_cast<int32_t*>(s->st[kApexQPa2]);
  a.replies = s->d_block + (size_t)s->num_envs * DRL_A3C_SERVER_REPORT_BYTES;
  a.T = s->T;
  DRL_CUDA_CHECK((launch_k(a3c_server_scatter_kernel, n, kThreads, 0, st, a)));
  return DRL_OK;
}

int server_init(drl_a3c_policy_server* s, void* exchange) {
  DRL_TRY(server_core_init(s, exchange));
  PolicyCore* h = s->engine;
  const size_t E = s->num_envs, MB = h->max_batch;
  DRL_TRY(dev_alloc(s, &s->tab.pa, E));
  DRL_TRY(dev_alloc(s, &s->tab.t, E, 0xff));   // -1: no step yet
  DRL_TRY(dev_alloc(s, &s->out_policy, MB * h->A));
  DRL_TRY(dev_alloc(s, &s->out_action, MB));
  DRL_TRY(dev_alloc(s, &s->out_prob, MB));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_a3c_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes) {
  if (!bytes) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (num_envs < 1 || num_envs > kServerMaxEnvs) {
    set_error("a3c policy server: num_envs must be in [1, %d] (got %d)", kServerMaxEnvs, num_envs);
    return DRL_ERR_INVALID;
  }
  *bytes = server_exchange_bytes(num_envs, DRL_A3C_SERVER_REPORT_BYTES);
  return DRL_OK;
}

int drl_a3c_policy_server_create(drl_a3c_policy* p, drl_a3c_queue* q, int32_t num_envs, void* exchange,
                                 int64_t exchange_size, drl_a3c_policy_server** out) {
  constexpr const char* kName = "a3c policy server";
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  if (!p) { set_error("null a3c policy handle"); return DRL_ERR_INVALID; }
  if (!q) { set_error("null a3c queue handle"); return DRL_ERR_INVALID; }
  DRL_TRY(server_check_block(kName, num_envs, DRL_A3C_SERVER_REPORT_BYTES, exchange, exchange_size));
  PolicyCore* h = apex_policy_core_of(p);
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (apex_policy_algo(p) != 1) {
    set_error("%s: this policy is Ape-X; an A3C policy server needs an A3C engine (algo 1)", kName);
    return DRL_ERR_INVALID;
  }
  if (q->device != h->device) {
    set_error("%s: the queue is on device %d, the policy on device %d", kName, q->device, h->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != h->A) {
    set_error("%s: the queue has num_action %d, the policy %d", kName, q->A, h->A);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:a3c_policy_server_create");
  drl_a3c_policy_server* s = new drl_a3c_policy_server();
  s->name = kName;
  s->serve_range = "drl:a3c_policy_server_serve";
  s->policy = p;
  s->engine = h;
  s->q = q;
  s->num_envs = num_envs;
  s->report_bytes = DRL_A3C_SERVER_REPORT_BYTES;
  s->T = q->T;
  s->enqueue_serve = enqueue_serve;
  int rc = server_check_queue_rows(s, "unrolls");
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

int drl_a3c_policy_server_destroy(drl_a3c_policy_server* s) { return server_destroy(s); }

int drl_a3c_policy_server_serve(drl_a3c_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms) {
  if (!s) { set_error("null a3c policy server handle"); return DRL_ERR_INVALID; }
  return server_serve(s, n, env_ids, timeout_ms);
}

}  // extern "C"
