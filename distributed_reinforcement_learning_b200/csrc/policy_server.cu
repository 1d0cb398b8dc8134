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
//   the engine's act kernels   (policy_enqueue_forward), outputs into device memory
//   server_scatter_kernel      step t of each row into the staging; h, c, previous action, t into the table; action
//                              and max probability into the row's reply record
// The commit's waits on the target slots' release events precede these on the stream, its commit events follow them,
// so one graph per n holds all four; a serve in which no row completes a trajectory replays a second graph of n
// without the commit kernel.
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "policy_core.cuh"
#include "traj_queue.cuh"

namespace drl {
namespace {

constexpr int kMaxEnvs = 256;
constexpr int kThreads = 256;
constexpr int kCommitSplit = 16;   // CTAs per committed trajectory (one trajectory is 0.6 MB at T = 20)

static_assert(DRL_SERVER_REPORT_FRAME == 0 && DRL_SERVER_REPORT_UNIFORM >= Geo::FRAME, "report layout");
static_assert(DRL_SERVER_REPORT_BYTES % 16 == 0 && DRL_SERVER_REPLY_BYTES % 16 == 0, "16-byte records");

// the device word block of one serve (int32): env ids [max_batch], completed-row count, then per completed row its
// environment, target slot and row
struct Words {
  int max_batch;
  size_t env() const { return 0; }
  size_t m() const { return (size_t)max_batch; }
  size_t commits() const { return (size_t)max_batch + 1; }
  size_t count() const { return (size_t)max_batch + 1 + 3 * (size_t)max_batch; }
};

struct Table {
  float* h;          // [num_envs][256]
  float* c;          // [num_envs][256]
  int32_t* pa;       // [num_envs]
  int32_t* t;        // [num_envs]: the step the next act records, -1 before the first
};

// staging / queue field pointers, in TrajField order
struct Fields {
  uint8_t* p[kTrajFields];
  size_t sz[kTrajFields];
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

// ---- queue_commit_rows_kernel -----------------------------------------------------------------------------------
// grid (n, kCommitSplit): CTA (j, k) copies part k of every field of completed row j (j < *m; the rest exit) from the
// staging of its environment to its reserved queue position.  16-byte copies where the field allows.
struct CommitArgs {
  const int32_t* m;          // completed-row count
  const int32_t* rows;       // [m][3]: environment, slot, row
  Fields src;                // staging field bases (record e at + e * sz)
  uint8_t* dst_base;         // queue slots
  size_t dst_off[kTrajFields];
  size_t slot_bytes;
};

__global__ void __launch_bounds__(kThreads) queue_commit_rows_kernel(const CommitArgs a) {
  kernel_prologue();
  const int j = blockIdx.x;
  if (j >= *a.m) return;
  const int e = a.rows[3 * j], slot = a.rows[3 * j + 1], qrow = a.rows[3 * j + 2];
  const int nthreads = kThreads * kCommitSplit, gtid = blockIdx.y * kThreads + threadIdx.x;
#pragma unroll 1
  for (int f = 0; f < kTrajFields; ++f) {
    const size_t sz = a.src.sz[f];
    const uint8_t* s = a.src.p[f] + (size_t)e * sz;
    uint8_t* d = a.dst_base + (size_t)slot * a.slot_bytes + a.dst_off[f] + (size_t)qrow * sz;
    if (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d) | sz) & 15) == 0) {
      const uint4* s4 = reinterpret_cast<const uint4*>(s);
      uint4* d4 = reinterpret_cast<uint4*>(d);
      for (size_t i = gtid; i < sz / 16; i += nthreads) d4[i] = s4[i];
    } else {
      for (size_t i = gtid; i < sz; i += nthreads) d[i] = s[i];
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

int64_t exchange_bytes(int num_envs) {
  return (int64_t)align_up((size_t)num_envs * (DRL_SERVER_REPORT_BYTES + DRL_SERVER_REPLY_BYTES), 4096);
}

}  // namespace
}  // namespace drl

using namespace drl;

struct drl_policy_server {
  drl_policy* policy = nullptr;
  PolicyCore* engine = nullptr;
  drl_traj_queue* q = nullptr;
  int num_envs = 0, T = 0;
  std::mutex mu;                      // one serve at a time
  uint8_t* host_block = nullptr;      // the caller's exchange block, registered while the server lives
  uint8_t* d_block = nullptr;         // its device alias
  Table tab{};
  Fields st{};                        // staging [num_envs] trajectories
  float* out_policy = nullptr;        // the act's outputs [max_batch][A] / [max_batch][256] / [max_batch]
  float *out_h = nullptr, *out_c = nullptr;
  int32_t* out_action = nullptr;
  Words words{};
  int32_t* d_words = nullptr;
  int32_t* h_words = nullptr;         // pinned
  std::vector<int> t;                 // host mirror of the table's t
  std::vector<cudaGraphExec_t> graphs[2];   // per n: [0] without the commit kernel (no row completes), [1] with it
  std::vector<void*> allocs;
};

namespace {

// the serve of n rows; `commit`: with queue_commit_rows_kernel (some row completes a trajectory)
int enqueue_serve(drl_policy_server* s, int n, bool commit) {
  PolicyCore* h = s->engine;
  cudaStream_t st = h->stream;
  DRL_CUDA_CHECK(cudaMemcpyAsync(s->d_words, s->h_words, s->words.count() * 4, cudaMemcpyHostToDevice, st));
  const PolicyInRows in = policy_input_rows(s->policy, n);
  const int32_t* env = s->d_words + s->words.env();
  GatherArgs g;
  g.reports = s->d_block;
  g.env = env;
  g.tab = s->tab;
  g.in = in;
  g.st_reward = reinterpret_cast<float*>(s->st.p[kTrajReward]);
  g.st_done = s->st.p[kTrajDone];
  g.T = s->T;
  DRL_CUDA_CHECK((launch_k(server_gather_kernel, n, kThreads, 0, st, g)));
  if (commit) {
    CommitArgs c;
    c.m = s->d_words + s->words.m();
    c.rows = s->d_words + s->words.commits();
    c.src = s->st;
    c.dst_base = s->q->base;
    for (int f = 0; f < kTrajFields; ++f) c.dst_off[f] = s->q->off[f];
    c.slot_bytes = s->q->slot_bytes;
    DRL_CUDA_CHECK((launch_k(queue_commit_rows_kernel, dim3(n, kCommitSplit), kThreads, 0, st, c)));
  }
  const PolicyOutRows out{s->out_policy, s->out_h, s->out_c, s->out_action};
  DRL_TRY(policy_enqueue_forward(s->policy, n, out));
  ScatterArgs a;
  a.env = env;
  a.in = in;
  a.out = out;
  a.tab = s->tab;
  a.st = s->st;
  a.replies = s->d_block + (size_t)s->num_envs * DRL_SERVER_REPORT_BYTES;
  a.T = s->T;
  a.A = h->A;
  DRL_CUDA_CHECK((launch_k(server_scatter_kernel, n, kThreads, 0, st, a)));
  return DRL_OK;
}

void release(drl_policy_server* s) {
  if (s->engine) {
    cudaSetDevice(s->engine->device);
    if (s->engine->stream) cudaStreamSynchronize(s->engine->stream);
  }
  for (auto& v : s->graphs)
    for (auto g : v) if (g) cudaGraphExecDestroy(g);
  for (void* p : s->allocs) cudaFree(p);
  if (s->h_words) cudaFreeHost(s->h_words);
  if (s->host_block) cudaHostUnregister(s->host_block);
  cudaGetLastError();
}

int server_init(drl_policy_server* s, void* exchange) {
  PolicyCore* h = s->engine;
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t E = s->num_envs, MB = h->max_batch;
  DRL_TRY(dev_alloc(s, &s->tab.h, E * Geo::L));
  DRL_TRY(dev_alloc(s, &s->tab.c, E * Geo::L));
  DRL_TRY(dev_alloc(s, &s->tab.pa, E));
  DRL_TRY(dev_alloc(s, &s->tab.t, E, 0xff));   // -1: no step yet
  for (int f = 0; f < kTrajFields; ++f) {
    s->st.sz[f] = s->q->sz[f];
    DRL_TRY(dev_alloc(s, &s->st.p[f], E * s->q->sz[f]));
  }
  DRL_TRY(dev_alloc(s, &s->out_policy, MB * h->A));
  DRL_TRY(dev_alloc(s, &s->out_h, MB * Geo::L));
  DRL_TRY(dev_alloc(s, &s->out_c, MB * Geo::L));
  DRL_TRY(dev_alloc(s, &s->out_action, MB));
  s->words.max_batch = (int)MB;
  DRL_TRY(dev_alloc(s, &s->d_words, s->words.count()));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&s->h_words, s->words.count() * 4, cudaHostAllocDefault));
  memset(s->h_words, 0, s->words.count() * 4);
  DRL_CUDA_CHECK(cudaHostRegister(exchange, (size_t)exchange_bytes(s->num_envs),
                                  cudaHostRegisterMapped | cudaHostRegisterPortable));
  s->host_block = static_cast<uint8_t*>(exchange);
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&s->d_block, exchange, 0));
  s->t.assign(E, -1);
  for (auto& v : s->graphs) v.assign(MB + 1, nullptr);
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes) {
  if (!bytes) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (num_envs < 1 || num_envs > kMaxEnvs) {
    set_error("policy server: num_envs must be in [1, %d] (got %d)", kMaxEnvs, num_envs);
    return DRL_ERR_INVALID;
  }
  *bytes = exchange_bytes(num_envs);
  return DRL_OK;
}

int drl_policy_server_create(drl_policy* p, drl_traj_queue* q, int32_t num_envs, void* exchange,
                             int64_t exchange_size, drl_policy_server** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  if (!p) { set_error("null policy handle"); return DRL_ERR_INVALID; }
  if (!q) { set_error("null trajectory queue handle"); return DRL_ERR_INVALID; }
  int64_t need = 0;
  DRL_TRY(drl_policy_server_exchange_bytes(num_envs, &need));
  const long page = sysconf(_SC_PAGESIZE);
  if (!exchange || reinterpret_cast<uintptr_t>(exchange) % (uintptr_t)page != 0) {
    set_error("policy server: the exchange block must be page-aligned (%ld bytes)", page);
    return DRL_ERR_INVALID;
  }
  if (exchange_size < need) {
    set_error("policy server: the exchange block has %lld bytes, %d environments need %lld", (long long)exchange_size,
              num_envs, (long long)need);
    return DRL_ERR_INVALID;
  }
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
  const int most = std::min(num_envs, h->max_batch);
  if (most > traj_queue_max_rows(q)) {
    set_error("policy server: one serve may commit %d trajectories, the queue takes at most %d at once", most,
              traj_queue_max_rows(q));
    return DRL_ERR_INVALID;
  }
  NvtxRange nv("drl:policy_server_create");
  drl_policy_server* s = new drl_policy_server();
  s->policy = p;
  s->engine = h;
  s->q = q;
  s->num_envs = num_envs;
  s->T = q->T;
  const int rc = server_init(s, exchange);
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    release(s);
    delete s;
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = s;
  return DRL_OK;
}

int drl_policy_server_destroy(drl_policy_server* s) {
  if (!s) return DRL_OK;
  {
    std::lock_guard<std::mutex> lk(s->mu);
    std::lock_guard<std::recursive_mutex> lk2(s->engine->mu);
    release(s);
  }
  delete s;
  return DRL_OK;
}

int drl_policy_server_serve(drl_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms) {
  if (!s) { set_error("null policy server handle"); return DRL_ERR_INVALID; }
  if (!env_ids) { set_error("policy server serve: null env_ids"); return DRL_ERR_INVALID; }
  PolicyCore* h = s->engine;
  if (n < 1 || n > h->max_batch) {
    set_error("policy server serve: n must be in [1, %d] (the engine's max_batch; got %d)", h->max_batch, n);
    return DRL_ERR_INVALID;
  }
  std::lock_guard<std::mutex> slk(s->mu);
  std::vector<char> seen(s->num_envs, 0);
  std::vector<int> done_rows;   // rows whose serve completes their staged trajectory
  for (int r = 0; r < n; ++r) {
    const int e = env_ids[r];
    if (e < 0 || e >= s->num_envs) {
      set_error("policy server serve: env_ids[%d] = %d is outside [0, %d)", r, e, s->num_envs);
      return DRL_ERR_INVALID;
    }
    if (seen[e]) { set_error("policy server serve: environment %d is listed twice", e); return DRL_ERR_INVALID; }
    seen[e] = 1;
    if (s->t[e] == 0) done_rows.push_back(r);
  }
  const int m = (int)done_rows.size();
  // reserve without the engine's lock: a learner thread may sync this engine while the serve waits for space
  std::vector<TrajSegment> segs;
  if (m > 0) DRL_TRY(traj_queue_reserve(s->q, m, timeout_ms, &segs));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  NvtxRange nv("drl:policy_server_serve");
  int32_t* w = s->h_words;   // free: the previous serve waited for the stream
  memcpy(w + s->words.env(), env_ids, (size_t)n * 4);
  w[s->words.m()] = m;
  int32_t* cw = w + s->words.commits();
  for (const TrajSegment& g : segs)
    for (int i = 0; i < g.rows; ++i) {
      const int j = g.src0 + i;
      cw[3 * j] = env_ids[done_rows[j]];
      cw[3 * j + 1] = g.slot;
      cw[3 * j + 2] = g.row0 + i;
    }
  cudaStream_t st = h->stream;
  const int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(h->device));
    for (const TrajSegment& g : segs) DRL_CUDA_CHECK(cudaStreamWaitEvent(st, g.ev_release, 0));
    const bool commit = m > 0;
    if (h->use_cuda_graph) {
      cudaGraphExec_t& graph = s->graphs[commit][n];
      if (!graph) {
        // this serve runs eagerly (the launchers set their attributes and tensor maps outside capture); the capture
        // only records, so the state table advances once
        DRL_TRY(enqueue_serve(s, n, commit));
        DRL_TRY(capture_graph(st, [&] { return enqueue_serve(s, n, commit); }, &graph));
      } else {
        DRL_CUDA_CHECK(cudaGraphLaunch(graph, st));
      }
    } else {
      DRL_TRY(enqueue_serve(s, n, commit));
    }
    for (const TrajSegment& g : segs) DRL_CUDA_CHECK(cudaEventRecord(g.ev_commit, st));
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    if (m > 0) traj_queue_fail(s->q, get_error());
    return rc;
  }
  if (m > 0) traj_queue_commit(s->q, segs);
  for (int r = 0; r < n; ++r) {
    int& t = s->t[env_ids[r]];
    t = (std::max(t, 0) + 1) % s->T;
  }
  DRL_CUDA_CHECK(cudaStreamSynchronize(st));
  return DRL_OK;
}

}  // extern "C"
