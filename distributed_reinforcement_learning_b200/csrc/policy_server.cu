// policy_server.cu -- the IMPALA policy server behind drl_policy_server_* (include/drl_b200.h; DESIGN.md section 16).
// One engine (policy.cu) serves environments that step in other processes.  Each environment's recurrent state lives
// in a device state table and its unfinished trajectory in a device staging indexed by environment; the processes
// exchange frames and actions with the server through a host block registered as mapped memory, which the kernels
// read and write directly.
//
// One serve of n rows = one upload of the call's word block (env ids, completed-row list) + on the engine's stream:
//   server_gather_kernel       report -> the engine's device input rows (frame, uniform; h, c, previous action from
//                              the table, or 0 on reset); the previous step's reward and done -> staging at t - 1
//   queue_commit_rows_kernel   the staged trajectories that step T-1 completed -> their reserved queue positions
//                              (server_core.cu)
//   the engine's act kernels   (policy_enqueue_forward), outputs into device memory
//   server_scatter_kernel      step t of each row into the staging; h, c, previous action, t into the table; action
//                              and max probability into the row's reply record
// The commit's waits on the target slots' release events precede these on the stream, its commit events follow them,
// so one graph per n holds all four; a serve in which no row completes a trajectory replays a second graph of n
// without the commit kernel.  The binding, the word block, the reservation and the graphs are the server core's
// (server_core.cuh).
#include "server_core.cuh"

namespace drl {
namespace {

constexpr int kThreads = kServerThreads;

static_assert(DRL_SERVER_REPORT_FRAME == 0 && DRL_SERVER_REPORT_UNIFORM >= Geo::FRAME, "report layout");

struct Table {
  float* h;          // [num_envs][256]
  float* c;          // [num_envs][256]
  int32_t* pa;       // [num_envs]
  int32_t* t;        // [num_envs]: the step the next act records, -1 before the first
};

// staging field pointers, in TrajField order
struct Fields {
  uint8_t* p[kTrajFields];
};

// ---- server_gather_kernel ---------------------------------------------------------------------------------------
struct GatherArgs {
  const uint8_t* reports;    // mapped exchange block
  const int32_t* env;        // [n]
  Table tab;
  PolicyInRows in;
  float* st_reward;          // staging [num_envs][T]
  uint8_t* st_done;          // [num_envs][T]
  int T;
};

__global__ void __launch_bounds__(kThreads) server_gather_kernel(const GatherArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  const uint8_t* rep = a.reports + (size_t)e * DRL_SERVER_REPORT_BYTES;
  // every load of the frame issued before the first store: each is a round trip over PCIe
  const uint4* f = reinterpret_cast<const uint4*>(rep + DRL_SERVER_REPORT_FRAME);
  uint4* fd = reinterpret_cast<uint4*>(a.in.frames + (size_t)row * Geo::FRAME);
  constexpr int kPer = (Geo::FRAME / 16 + kThreads - 1) / kThreads;
  uint4 v[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < Geo::FRAME / 16) v[k] = f[tid + k * kThreads];
#pragma unroll
  for (int k = 0; k < kPer; ++k) if (tid + k * kThreads < Geo::FRAME / 16) fd[tid + k * kThreads] = v[k];
  // one 16-byte load per scalar field of the report
  const bool reset = reinterpret_cast<const uint4*>(rep + DRL_SERVER_REPORT_RESET)->x & 0xffu;
  if (tid < Geo::L / 4) {
    const float4 x = reset ? zero4() : reinterpret_cast<const float4*>(a.tab.h + (size_t)e * Geo::L)[tid];
    reinterpret_cast<float4*>(a.in.h0 + (size_t)row * Geo::L)[tid] = x;
  } else if (tid < Geo::L / 2) {
    const int i = tid - Geo::L / 4;
    const float4 x = reset ? zero4() : reinterpret_cast<const float4*>(a.tab.c + (size_t)e * Geo::L)[i];
    reinterpret_cast<float4*>(a.in.c0 + (size_t)row * Geo::L)[i] = x;
  } else if (tid == Geo::L / 2) {
    a.in.pa[row] = reset ? 0 : a.tab.pa[e];
  } else if (tid == Geo::L / 2 + 1) {
    const uint4 u = *reinterpret_cast<const uint4*>(rep + DRL_SERVER_REPORT_UNIFORM);
    a.in.uniform[row] = __hiloint2double((int)u.y, (int)u.x);
  } else if (tid == Geo::L / 2 + 2) {
    const int t = a.tab.t[e];
    if (t >= 0) {   // the reward and done of the previous step (t - 1, or T - 1 of the unroll step t = 0 follows)
      const size_t prev = (size_t)e * a.T + (t + a.T - 1) % a.T;
      const uint4 r = *reinterpret_cast<const uint4*>(rep + DRL_SERVER_REPORT_REWARD);
      const uint4 d = *reinterpret_cast<const uint4*>(rep + DRL_SERVER_REPORT_DONE);
      a.st_reward[prev] = __uint_as_float(r.x);
      a.st_done[prev] = (uint8_t)(d.x & 0xffu);
    }
  }
}

// ---- server_scatter_kernel --------------------------------------------------------------------------------------
struct ScatterArgs {
  const int32_t* env;        // [n]
  PolicyInRows in;           // what the act read
  PolicyOutRows out;         // what it computed (device)
  Table tab;
  Fields st;                 // staging
  uint8_t* replies;          // mapped reply records
  int T, A;
};

__global__ void __launch_bounds__(kThreads) server_scatter_kernel(const ScatterArgs a) {
  kernel_prologue();
  const int row = blockIdx.x, tid = threadIdx.x;
  const int e = a.env[row];
  // every thread reads the step before the barrier below; the table's step is written only after it
  const int t = max(a.tab.t[e], 0);
  const size_t dst = (size_t)e * a.T + t;
  const uint4* f = reinterpret_cast<const uint4*>(a.in.frames + (size_t)row * Geo::FRAME);
  uint4* fd = reinterpret_cast<uint4*>(a.st.p[kTrajState] + dst * Geo::FRAME);
  for (int i = tid; i < Geo::FRAME / 16; i += kThreads) fd[i] = f[i];
  float* sh = reinterpret_cast<float*>(a.st.p[kTrajH]) + dst * Geo::L;
  float* sc = reinterpret_cast<float*>(a.st.p[kTrajC]) + dst * Geo::L;
  if (tid < Geo::L / 4) {
    reinterpret_cast<float4*>(sh)[tid] = reinterpret_cast<const float4*>(a.in.h0 + (size_t)row * Geo::L)[tid];
    reinterpret_cast<float4*>(a.tab.h + (size_t)e * Geo::L)[tid] =
        reinterpret_cast<const float4*>(a.out.h1 + (size_t)row * Geo::L)[tid];
  } else if (tid < Geo::L / 2) {
    const int i = tid - Geo::L / 4;
    reinterpret_cast<float4*>(sc)[i] = reinterpret_cast<const float4*>(a.in.c0 + (size_t)row * Geo::L)[i];
    reinterpret_cast<float4*>(a.tab.c + (size_t)e * Geo::L)[i] =
        reinterpret_cast<const float4*>(a.out.c1 + (size_t)row * Geo::L)[i];
  } else if (tid < Geo::L / 2 + 32) {
    // warp 4: the policy row into the staging, its maximum and the action into the reply, the table's pa
    const int lane = tid & 31;
    const float p = lane < a.A ? a.out.policy[(size_t)row * a.A + lane] : -INFINITY;
    if (lane < a.A) reinterpret_cast<float*>(a.st.p[kTrajMu])[dst * a.A + lane] = p;
    const float mx = warp_max(p);
    if (lane == 0) {
      const int32_t act = a.out.action[row];
      reinterpret_cast<int32_t*>(a.st.p[kTrajPa])[dst] = a.in.pa[row];
      reinterpret_cast<int32_t*>(a.st.p[kTrajAction])[dst] = act;
      a.tab.pa[e] = act;
      uint8_t* rep = a.replies + (size_t)e * DRL_SERVER_REPLY_BYTES;
      *reinterpret_cast<int32_t*>(rep + DRL_SERVER_REPLY_ACTION) = act;
      *reinterpret_cast<float*>(rep + DRL_SERVER_REPLY_MAX_PROB) = mx;
    }
  }
  __syncthreads();
  if (tid == 0) a.tab.t[e] = (t + 1) % a.T;
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_policy_server : ServerCore {
  drl_policy* policy = nullptr;
  Table tab{};
  float* out_policy = nullptr;        // the act's outputs [max_batch][A] / [max_batch][256] / [max_batch]
  float *out_h = nullptr, *out_c = nullptr;
  int32_t* out_action = nullptr;
};

namespace {

// the serve of n rows; `commit`: with queue_commit_rows_kernel (some row completes a trajectory)
int enqueue_serve(ServerCore* core, int n, bool commit) {
  drl_policy_server* s = static_cast<drl_policy_server*>(core);
  PolicyCore* h = s->engine;
  cudaStream_t st = h->stream;
  DRL_TRY(server_upload_words(s));
  const PolicyInRows in = policy_input_rows(s->policy, n);
  const int32_t* env = s->d_words + s->words.env();
  Fields fields;
  for (int f = 0; f < kTrajFields; ++f) fields.p[f] = s->st[f];
  GatherArgs g;
  g.reports = s->d_block;
  g.env = env;
  g.tab = s->tab;
  g.in = in;
  g.st_reward = reinterpret_cast<float*>(s->st[kTrajReward]);
  g.st_done = s->st[kTrajDone];
  g.T = s->T;
  DRL_CUDA_CHECK((launch_k(server_gather_kernel, n, kThreads, 0, st, g)));
  if (commit) DRL_TRY(server_enqueue_commit(s, n));
  const PolicyOutRows out{s->out_policy, s->out_h, s->out_c, s->out_action};
  DRL_TRY(policy_enqueue_forward(s->policy, n, out));
  ScatterArgs a;
  a.env = env;
  a.in = in;
  a.out = out;
  a.tab = s->tab;
  a.st = fields;
  a.replies = s->d_block + (size_t)s->num_envs * DRL_SERVER_REPORT_BYTES;
  a.T = s->T;
  a.A = h->A;
  DRL_CUDA_CHECK((launch_k(server_scatter_kernel, n, kThreads, 0, st, a)));
  return DRL_OK;
}

int server_init(drl_policy_server* s, void* exchange) {
  DRL_TRY(server_core_init(s, exchange));
  PolicyCore* h = s->engine;
  const size_t E = s->num_envs, MB = h->max_batch;
  DRL_TRY(dev_alloc(s, &s->tab.h, E * Geo::L));
  DRL_TRY(dev_alloc(s, &s->tab.c, E * Geo::L));
  DRL_TRY(dev_alloc(s, &s->tab.pa, E));
  DRL_TRY(dev_alloc(s, &s->tab.t, E, 0xff));   // -1: no step yet
  DRL_TRY(dev_alloc(s, &s->out_policy, MB * h->A));
  DRL_TRY(dev_alloc(s, &s->out_h, MB * Geo::L));
  DRL_TRY(dev_alloc(s, &s->out_c, MB * Geo::L));
  DRL_TRY(dev_alloc(s, &s->out_action, MB));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_policy_server_create(drl_policy* p, drl_traj_queue* q, int32_t num_envs, void* exchange,
                             int64_t exchange_size, drl_policy_server** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  if (!p) { set_error("null policy handle"); return DRL_ERR_INVALID; }
  if (!q) { set_error("null trajectory queue handle"); return DRL_ERR_INVALID; }
  DRL_TRY(server_check_block("policy server", num_envs, DRL_SERVER_REPORT_BYTES, exchange, exchange_size));
  PolicyCore* h = policy_core_of(p);
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (q->device != h->device) {
    set_error("policy server: the queue is on device %d, the policy on device %d", q->device, h->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != h->A) { set_error("policy server: the queue has num_action %d, the policy %d", q->A, h->A); return DRL_ERR_INVALID; }
  if (q->H != Geo::IH || q->W != Geo::IW || q->C != Geo::IC || q->L != Geo::L) {
    set_error("policy server: the queue stores %dx%dx%d frames and lstm %d, the policy takes %dx%dx%d and %d", q->H,
              q->W, q->C, q->L, Geo::IH, Geo::IW, Geo::IC, Geo::L);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:policy_server_create");
  drl_policy_server* s = new drl_policy_server();
  s->name = "policy server";
  s->serve_range = "drl:policy_server_serve";
  s->policy = p;
  s->engine = h;
  s->q = q;
  s->num_envs = num_envs;
  s->report_bytes = DRL_SERVER_REPORT_BYTES;
  s->T = q->T;
  s->enqueue_serve = enqueue_serve;
  int rc = server_check_queue_rows(s, "trajectories");
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

int drl_policy_server_destroy(drl_policy_server* s) { return server_destroy(s); }

int drl_policy_server_serve(drl_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms) {
  if (!s) { set_error("null policy server handle"); return DRL_ERR_INVALID; }
  return server_serve(s, n, env_ids, timeout_ms);
}

}  // extern "C"
