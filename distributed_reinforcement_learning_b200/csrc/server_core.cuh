// server_core.cuh -- the part of a policy server (DESIGN.md sections 16 and 17) that depends neither on the engine's
// network nor on what one queue record is: the binding of one engine to one device queue and to an exchange block the
// caller shares with the processes that step the environments, the registration of that block, the per-serve word
// block (pinned + device), the host mirror of each environment's step t, the env-id checks, the queue reservation
// around a serve, the graph pair per n, and queue_commit_rows_kernel.  The IMPALA server (policy_server.cu:
// drl_policy_server) and the R2D2 server (r2d2_policy_server.cu: drl_r2d2_policy_server) derive from ServerCore; each
// adds its state table, its gather and scatter kernels and its enqueue of one serve.
//
// The IMPALA and R2D2 families use the same record sizes and stride in the exchange block (DRL_SERVER_REPORT_BYTES /
// DRL_SERVER_REPLY_BYTES), so one drl_policy_server_exchange_bytes sizes the block of either.  The A3C server
// (a3c_policy_server.cu: drl_a3c_policy_server) reports two frames per environment, so each family sets its report
// size (ServerCore::report_bytes); every family's reply record is DRL_SERVER_REPLY_BYTES.
#pragma once
#include <mutex>
#include <vector>

#include "policy_core.cuh"
#include "traj_queue.cuh"

namespace drl {

constexpr int kServerMaxEnvs = 256;
constexpr int kServerThreads = 256;

// the device word block of one serve (int32): env ids [max_batch], completed-row count, per completed row its
// environment, target slot and row [max_batch][3], then `extra` [max_batch] words per row the family stages
// (stage_rows below)
struct ServerWords {
  int max_batch = 0, extra = 0;
  size_t env() const { return 0; }
  size_t m() const { return (size_t)max_batch; }
  size_t commits() const { return (size_t)max_batch + 1; }
  size_t extra_words() const { return (size_t)max_batch + 1 + 3 * (size_t)max_batch; }
  size_t count() const { return extra_words() + (size_t)extra * max_batch; }
};

struct ServerCore {
  // Enqueues the serve of the n rows staged in the word block on the engine's stream (after the upload of the word
  // block, which server_upload_words enqueues); `commit`: with server_enqueue_commit (some row completes a record).
  using EnqueueServe = int (*)(ServerCore* s, int n, bool commit);
  // Checks and stages what the family reads from the reports on the host (into the word block's extra words) for the
  // n rows env_ids, before anything else of the serve happens; may be null.
  using StageRows = int (*)(ServerCore* s, int n, const int32_t* env_ids);

  // set by the family before server_core_init
  const char* name = "policy server";       // "<name> serve: ..." in error messages
  const char* serve_range = "drl:policy_server_serve";
  PolicyCore* engine = nullptr;
  QueueCore* q = nullptr;
  int num_envs = 0, T = 0;                  // environments, steps per record
  EnqueueServe enqueue_serve = nullptr;
  StageRows stage_rows = nullptr;
  int extra_words = 0;
  int report_bytes = 0;                     // stride of the report records; the replies follow num_envs of them

  std::mutex mu;                            // one serve at a time
  uint8_t* host_block = nullptr;            // the caller's exchange block, registered while the server lives
  uint8_t* d_block = nullptr;               // its device alias
  uint8_t* st[kQueueMaxFields] = {};        // staging: field f of environment e's record at st[f] + e * q->sz[f]
  ServerWords words{};
  int32_t* d_words = nullptr;
  int32_t* h_words = nullptr;               // pinned
  std::vector<int> t;                       // host mirror of the state table's t (-1 before the first act)
  std::vector<cudaGraphExec_t> graphs[2];   // per n: [0] without the commit kernel (no row completes), [1] with it
  std::vector<void*> allocs;
};

// num_envs * (report_bytes + DRL_SERVER_REPLY_BYTES) rounded up to a page
int64_t server_exchange_bytes(int num_envs, int report_bytes);
// create's checks of the block, in this order: num_envs in [1, 256], a page-aligned block of at least
// server_exchange_bytes(num_envs, report_bytes) bytes (DRL_ERR_INVALID, "<name>: ...")
int server_check_block(const char* name, int num_envs, int report_bytes, const void* exchange, int64_t exchange_size);
// "one serve may commit min(num_envs, max_batch) records, the queue takes at most ..." (DRL_ERR_INVALID)
int server_check_queue_rows(const ServerCore* s, const char* records);
// Allocates the staging (one record per environment in the queue's field order), the word block and the host mirror
// of t, and registers the exchange block's server_exchange_bytes(num_envs, report_bytes) (mapped, portable) on the
// engine's device.  On failure the caller releases
// the server (server_core_release), keeping the error message.
int server_core_init(ServerCore* s, void* exchange);
// waits for the engine's stream, destroys the graphs, frees what server_core_init and dev_alloc made and unregisters
// the block (the caller holds the serve lock and the engine's lock)
void server_core_release(ServerCore* s);
// the serve's upload of its word block, on the engine's stream
int server_upload_words(ServerCore* s);
// queue_commit_rows_kernel over the completed rows of the word block (the staged records -> their reserved positions)
int server_enqueue_commit(ServerCore* s, int n);
// The serve of n rows: the env-id checks (each in [0, num_envs), no duplicate), the family's stage_rows, then the
// reservation of one queue position per row whose step T-1 this serve completes (without the engine's lock), and under
// the engine's lock the word block, the waits for the target slots' release events, enqueue_serve eagerly or through
// the graph of (n, commit), the commit events and a wait for the stream.  Advances the host mirror of t.  A failure
// after the reservation puts the queue into its failed state (traj_queue_fail).
int server_serve(ServerCore* s, int n, const int32_t* env_ids, int timeout_ms);

template <class S>
int server_destroy(S* s) {
  if (!s) return DRL_OK;
  {
    std::lock_guard<std::mutex> lk(s->mu);
    std::lock_guard<std::recursive_mutex> lk2(s->engine->mu);
    server_core_release(s);
  }
  delete s;
  return DRL_OK;
}

}  // namespace drl
