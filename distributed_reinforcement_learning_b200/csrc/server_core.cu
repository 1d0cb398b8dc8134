// server_core.cu -- the family-independent half of the policy servers (server_core.cuh; DESIGN.md sections 16, 17):
// the exchange block's size, create's shared checks, the registration of the block, the word block, the queue
// reservation around a serve, the graph pair per n, and queue_commit_rows_kernel, which serves every queue type.
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <string>

#include "server_core.cuh"

namespace drl {
namespace {

constexpr int kCommitSplit = 16;   // CTAs per committed record (one IMPALA trajectory is 0.6 MB at T = 20)

static_assert(DRL_SERVER_REPORT_BYTES % 16 == 0 && DRL_SERVER_REPLY_BYTES % 16 == 0, "16-byte records");

// ---- queue_commit_rows_kernel -----------------------------------------------------------------------------------
// grid (n, kCommitSplit): CTA (j, k) copies part k of every field of completed row j (j < *m; the rest exit) from the
// staging of its environment to its reserved queue position.  The fields are the queue's (QueueCore: nfields, sz,
// off), so one kernel serves the IMPALA trajectory queue and the R2D2 sequence queue.  16-byte copies where the field
// allows.
struct CommitArgs {
  const int32_t* m;                 // completed-row count
  const int32_t* rows;              // [m][3]: environment, slot, row
  const uint8_t* src[kQueueMaxFields];   // staging field bases (record e at + e * sz)
  size_t sz[kQueueMaxFields];
  size_t dst_off[kQueueMaxFields];
  uint8_t* dst_base;                // queue slots
  size_t slot_bytes;
  int nfields;
};

__global__ void __launch_bounds__(kServerThreads) queue_commit_rows_kernel(const CommitArgs a) {
  kernel_prologue();
  const int j = blockIdx.x;
  if (j >= *a.m) return;
  const int e = a.rows[3 * j], slot = a.rows[3 * j + 1], qrow = a.rows[3 * j + 2];
  const int nthreads = kServerThreads * kCommitSplit, gtid = blockIdx.y * kServerThreads + threadIdx.x;
#pragma unroll 1
  for (int f = 0; f < a.nfields; ++f) {
    const size_t sz = a.sz[f];
    const uint8_t* s = a.src[f] + (size_t)e * sz;
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

}  // namespace

int64_t server_exchange_bytes(int num_envs, int report_bytes) {
  return (int64_t)align_up((size_t)num_envs * ((size_t)report_bytes + DRL_SERVER_REPLY_BYTES), 4096);
}

int server_check_block(const char* name, int num_envs, int report_bytes, const void* exchange, int64_t exchange_size) {
  if (num_envs < 1 || num_envs > kServerMaxEnvs) {
    set_error("%s: num_envs must be in [1, %d] (got %d)", name, kServerMaxEnvs, num_envs);
    return DRL_ERR_INVALID;
  }
  const int64_t need = server_exchange_bytes(num_envs, report_bytes);
  const long page = sysconf(_SC_PAGESIZE);
  if (!exchange || reinterpret_cast<uintptr_t>(exchange) % (uintptr_t)page != 0) {
    set_error("%s: the exchange block must be page-aligned (%ld bytes)", name, page);
    return DRL_ERR_INVALID;
  }
  if (exchange_size < need) {
    set_error("%s: the exchange block has %lld bytes, %d environments need %lld", name, (long long)exchange_size,
              num_envs, (long long)need);
    return DRL_ERR_INVALID;
  }
  return DRL_OK;
}

int server_check_queue_rows(const ServerCore* s, const char* records) {
  const int most = std::min(s->num_envs, s->engine->max_batch);
  if (most > traj_queue_max_rows(s->q)) {
    set_error("%s: one serve may commit %d %s, the queue takes at most %d at once", s->name, most, records,
              traj_queue_max_rows(s->q));
    return DRL_ERR_INVALID;
  }
  return DRL_OK;
}

int server_core_init(ServerCore* s, void* exchange) {
  PolicyCore* h = s->engine;
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  const size_t E = s->num_envs, MB = h->max_batch;
  for (int f = 0; f < s->q->nfields; ++f) DRL_TRY(dev_alloc(s, &s->st[f], E * s->q->sz[f]));
  s->words.max_batch = (int)MB;
  s->words.extra = s->extra_words;
  DRL_TRY(dev_alloc(s, &s->d_words, s->words.count()));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&s->h_words, s->words.count() * 4, cudaHostAllocDefault));
  memset(s->h_words, 0, s->words.count() * 4);
  DRL_CUDA_CHECK(cudaHostRegister(exchange, (size_t)server_exchange_bytes(s->num_envs, s->report_bytes),
                                  cudaHostRegisterMapped | cudaHostRegisterPortable));
  s->host_block = static_cast<uint8_t*>(exchange);
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&s->d_block, exchange, 0));
  s->t.assign(E, -1);
  for (auto& v : s->graphs) v.assign(MB + 1, nullptr);
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

void server_core_release(ServerCore* s) {
  if (s->engine) {
    cudaSetDevice(s->engine->device);
    if (s->engine->stream) cudaStreamSynchronize(s->engine->stream);
  }
  for (auto& v : s->graphs)
    for (auto g : v) if (g) cudaGraphExecDestroy(g);
  for (void* p : s->allocs) cudaFree(p);
  s->allocs.clear();
  if (s->h_words) cudaFreeHost(s->h_words);
  s->h_words = nullptr;
  if (s->host_block) cudaHostUnregister(s->host_block);
  s->host_block = nullptr;
  cudaGetLastError();
}

int server_upload_words(ServerCore* s) {
  DRL_CUDA_CHECK(cudaMemcpyAsync(s->d_words, s->h_words, s->words.count() * 4, cudaMemcpyHostToDevice,
                                 s->engine->stream));
  return DRL_OK;
}

int server_enqueue_commit(ServerCore* s, int n) {
  const QueueCore* q = s->q;
  CommitArgs c;
  c.m = s->d_words + s->words.m();
  c.rows = s->d_words + s->words.commits();
  for (int f = 0; f < kQueueMaxFields; ++f) {
    const bool used = f < q->nfields;
    c.src[f] = used ? s->st[f] : nullptr;
    c.sz[f] = used ? q->sz[f] : 0;
    c.dst_off[f] = used ? q->off[f] : 0;
  }
  c.dst_base = q->base;
  c.slot_bytes = q->slot_bytes;
  c.nfields = q->nfields;
  DRL_CUDA_CHECK((launch_k(queue_commit_rows_kernel, dim3(n, kCommitSplit), kServerThreads, 0, s->engine->stream, c)));
  return DRL_OK;
}

int server_serve(ServerCore* s, int n, const int32_t* env_ids, int timeout_ms) {
  if (!env_ids) { set_error("%s serve: null env_ids", s->name); return DRL_ERR_INVALID; }
  PolicyCore* h = s->engine;
  if (n < 1 || n > h->max_batch) {
    set_error("%s serve: n must be in [1, %d] (the engine's max_batch; got %d)", s->name, h->max_batch, n);
    return DRL_ERR_INVALID;
  }
  std::lock_guard<std::mutex> slk(s->mu);
  std::vector<char> seen(s->num_envs, 0);
  std::vector<int> done_rows;   // rows whose serve completes their staged record
  for (int r = 0; r < n; ++r) {
    const int e = env_ids[r];
    if (e < 0 || e >= s->num_envs) {
      set_error("%s serve: env_ids[%d] = %d is outside [0, %d)", s->name, r, e, s->num_envs);
      return DRL_ERR_INVALID;
    }
    if (seen[e]) { set_error("%s serve: environment %d is listed twice", s->name, e); return DRL_ERR_INVALID; }
    seen[e] = 1;
    if (s->t[e] == 0) done_rows.push_back(r);
  }
  // the word block is free: the previous serve waited for the stream
  if (s->stage_rows) DRL_TRY(s->stage_rows(s, n, env_ids));
  const int m = (int)done_rows.size();
  // reserve without the engine's lock: a learner thread may sync this engine while the serve waits for space
  std::vector<TrajSegment> segs;
  if (m > 0) DRL_TRY(traj_queue_reserve(s->q, m, timeout_ms, &segs));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  NvtxRange nv(s->serve_range);
  int32_t* w = s->h_words;
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
        DRL_TRY(s->enqueue_serve(s, n, commit));
        DRL_TRY(capture_graph(st, [&] { return s->enqueue_serve(s, n, commit); }, &graph));
      } else {
        DRL_CUDA_CHECK(cudaGraphLaunch(graph, st));
      }
    } else {
      DRL_TRY(s->enqueue_serve(s, n, commit));
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

}  // namespace drl

using namespace drl;

extern "C" {

int drl_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes) {
  if (!bytes) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (num_envs < 1 || num_envs > kServerMaxEnvs) {
    set_error("policy server: num_envs must be in [1, %d] (got %d)", kServerMaxEnvs, num_envs);
    return DRL_ERR_INVALID;
  }
  *bytes = server_exchange_bytes(num_envs, DRL_SERVER_REPORT_BYTES);
  return DRL_OK;
}

}  // extern "C"
