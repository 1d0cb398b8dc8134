// traj_queue.cuh -- the device-resident queues (DESIGN.md sections 12 to 15): the FIFO core they share, the IMPALA
// trajectory queue (drl_traj_queue), the R2D2 sequence queue (drl_r2d2_queue), the Ape-X transition queue
// (drl_apex_queue) and the A3C trajectory queue (drl_a3c_queue), all in traj_queue.cu.  The producers are policy-engine
// recorders (queue_recorder.cuh) and the Ape-X actor buffers (apex_actor_buffer.cu); the consumers are
// drl_learner_stage_from_queue (learner.cu), drl_r2d2_replay_add_from_queue (r2d2_replay.cu),
// drl_apex_replay_add_from_queue (apex_replay.cu) and drl_a3c_stage_from_queue (apex.cu).
//
// The FIFO of drl_ring (ring.cu) with its batch slots in HBM instead of pinned host memory.  A slot holds `batch` records
// field-major, each field batch-major (`sz[f]` bytes per record), in the consumer's layout: the learner staging slot's
// (kernels.h: Inputs) for IMPALA, R2SeqRows / R2In (r2d2_replay.cu, r2d2_defs.cuh) for R2D2, ApexIn (apex_defs.cuh) of
// n = T rows for Ape-X and A3C (batch 1).  Queue position P (0, 1, 2, ... in reservation order) is row P % batch of slot
// (P / batch) % nslots.
//
// Ordering across streams, all through events the queue owns:
//   commit  (engine stream)     waits for ev_release of every slot it writes, copies, records one ev_commit per slot
//   pop     (consumer stream)   waits for every ev_commit of the popped slot, reads it, records the slot's ev_release
// Host-side state is guarded by `mu`; nobody holds it across a blocking wait on another handle's lock.
#pragma once
#include <condition_variable>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace drl {

// field order of an IMPALA slot (and of its recorders' staging): the ring's
enum TrajField { kTrajState = 0, kTrajReward, kTrajDone, kTrajMu, kTrajAction, kTrajPa, kTrajH, kTrajC, kTrajFields };
// field order of an R2D2 slot (and of its recorders' staging): R2SeqRows'
enum R2QueueField { kR2QFrames = 0, kR2QPa, kR2QAction, kR2QH, kR2QC, kR2QReward, kR2QDone, kR2QFields };
// field order of an Ape-X or A3C slot: ApexIn's (frames [2T]: state rows, then next_state rows; pa2 [2T]: previous_action, then
// action; reward [T]; done [T])
enum ApexQueueField { kApexQFrames = 0, kApexQPa2, kApexQReward, kApexQDone, kApexQFields };
// the largest T of an Ape-X queue: a push passes its T ring rows to the gather kernel by value
constexpr int kApexQueueMaxT = 512;
constexpr int kQueueMaxFields = 8;

// the rows [row0, row0 + rows) of `slot` that one commit writes, from its staging rows [src0, src0 + rows)
struct TrajSegment {
  int slot, row0, rows, src0;
  cudaEvent_t ev_commit;    // recorded by the committing engine once its copies into this slot are enqueued
  cudaEvent_t ev_release;   // the slot's previous consumer is done reading it
};

// the state of a queue that does not depend on what one record is
struct QueueCore {
  // names the queue in error messages: "<name> commit: ...", "<name> <pop_verb>: timed out (fewer than batch <items>
  // queued)"
  const char* name = "queue";
  const char* pop_verb = "pop";
  const char* items = "records";
  int nfields = 0, batch = 0, nslots = 0, device = 0;
  size_t sz[kQueueMaxFields] = {};    // bytes of one record per field
  size_t off[kQueueMaxFields] = {};   // field offsets inside a slot
  size_t slot_bytes = 0;
  uint8_t* base = nullptr;            // nslots * slot_bytes of device memory
  struct Slot {
    int reserved = 0, committed = 0;
    bool held = false;                // popped by a consumer, its reads not yet enqueued
    std::vector<cudaEvent_t> ev_commit;   // [batch]: the first n_commit belong to the commits since the last release
    int n_commit = 0;
    cudaEvent_t ev_release = nullptr;
  };
  std::vector<Slot> st;
  long long reserved_total = 0, committed_total = 0, popped_total = 0;
  bool failed = false;                // a commit failed after reserving its positions (traj_queue_fail)
  std::string failure;
  std::mutex mu;
  std::condition_variable cv_space, cv_ready;

  uint8_t* field(int slot, int f) { return base + (size_t)slot * slot_bytes + off[f]; }
};

}  // namespace drl

struct drl_traj_queue : drl::QueueCore {
  int T = 0, H = 0, W = 0, C = 0, A = 0, L = 0;
};

struct drl_r2d2_queue : drl::QueueCore {
  int S = 0, C = 1, A = 0;
  size_t frame = 0;                   // bytes of one 84x84xC frame
};

struct drl_apex_queue : drl::QueueCore {
  int T = 0, A = 0;                   // transitions per record, num_action
};

// the same record as drl_apex_queue (one actor unroll of T steps), a distinct type so that neither handle is accepted
// where the other is expected
struct drl_a3c_queue : drl::QueueCore {
  int T = 0, A = 0;                   // steps per record, num_action
};

namespace drl {

// Sets the queue's fields (nfields sizes sz, bytes per record), batch, device and nslots (capacity rounded up as the
// ring's plus one slot), then allocates and zeroes the slots and makes their events.  On failure the caller releases
// the queue (queue_core_release), keeping the error message.
int queue_core_init(QueueCore* q, int nfields, const size_t* sz, int capacity, int batch, int device);
// waits for every commit and release, frees the slots and events
void queue_core_release(QueueCore* q);
// committed minus popped
int queue_size(QueueCore* q);
// Synchronous copy of the k-th queued record (0 = the next to be popped): field f into dst[f], sz[f] bytes.
int queue_read(QueueCore* q, int k, void* const* dst);

// Producer side.  Reserves n consecutive positions, blocking while they are not free (timeout_ms < 0: forever;
// DRL_ERR_TIMEOUT with nothing changed otherwise).  Fills `segs` with the slots they fall in; the caller enqueues its
// copies, records each segment's ev_commit on its stream, then calls traj_queue_commit.  DRL_ERR_INVALID when n
// positions can never be free at once in this queue.
int traj_queue_reserve(QueueCore* q, int n, int timeout_ms, std::vector<TrajSegment>* segs);
void traj_queue_commit(QueueCore* q, const std::vector<TrajSegment>& segs);
// A commit that reserved positions and then could not enqueue its copies: the positions can never be filled, so the
// queue stops instead of blocking forever.  Wakes every waiter; from then on reserve, pop and read fail with
// DRL_ERR_STATE and `why` in the message.
void traj_queue_fail(QueueCore* q, const char* why);
// the largest n traj_queue_reserve can ever satisfy
int traj_queue_max_rows(const QueueCore* q);

// Consumer side.  Pops the oldest full batch slot (blocking like drl_ring_pop_batch) and returns its commit events;
// traj_queue_release then records the slot's ev_release on `s` (after the caller's reads of it) and hands it back to
// producers.
int traj_queue_pop(QueueCore* q, int timeout_ms, int* slot, std::vector<cudaEvent_t>* ev_commit);
int traj_queue_release(QueueCore* q, int slot, cudaStream_t s);

}  // namespace drl
