// traj_queue.cuh -- the device-resident IMPALA trajectory queue (DESIGN.md section 12): the state shared by its
// C-ABI (traj_queue.cu), the policy engine's recorder (policy.cu, the producer side) and the learner's
// drl_learner_stage_from_queue (learner.cu, the consumer side).
//
// The FIFO of drl_ring (ring.cu) with its batch slots in HBM instead of pinned host memory.  A slot holds `batch`
// trajectories field-major, each field in the batch-major layout of a learner staging slot (kernels.h: Inputs), so a
// popped batch is staged with eight contiguous device-to-device copies.  Queue position P (0, 1, 2, ... in reservation
// order) is row P % batch of slot (P / batch) % nslots.
//
// Ordering across streams, all through events the queue owns:
//   commit  (engine stream)   waits for ev_release of every slot it writes, copies, records one ev_commit per slot
//   stage   (learner copy)    waits for every ev_commit of the popped slot, copies, records the slot's ev_release
// Host-side state is guarded by `mu`; nobody holds it across a blocking wait on another handle's lock.
#pragma once
#include <condition_variable>
#include <mutex>
#include <string>
#include <vector>

#include "common.cuh"

namespace drl {

// field order of a slot (and of a recorder's staging): the ring's
enum TrajField { kTrajState = 0, kTrajReward, kTrajDone, kTrajMu, kTrajAction, kTrajPa, kTrajH, kTrajC, kTrajFields };

// the rows [row0, row0 + rows) of `slot` that one commit writes, from its staging rows [src0, src0 + rows)
struct TrajSegment {
  int slot, row0, rows, src0;
  cudaEvent_t ev_commit;    // recorded by the committing engine once its copies into this slot are enqueued
  cudaEvent_t ev_release;   // the slot's previous consumer is done reading it
};

}  // namespace drl

struct drl_traj_queue {
  int T = 0, H = 0, W = 0, C = 0, A = 0, L = 0, batch = 0, nslots = 0, device = 0;
  size_t sz[drl::kTrajFields] = {};    // bytes of one trajectory per field
  size_t off[drl::kTrajFields] = {};   // field offsets inside a slot
  size_t slot_bytes = 0;
  uint8_t* base = nullptr;             // nslots * slot_bytes of device memory
  struct Slot {
    int reserved = 0, committed = 0;
    bool held = false;                 // popped by a learner, its copies not yet enqueued
    std::vector<cudaEvent_t> ev_commit;   // [batch]: the first n_commit belong to the commits since the last release
    int n_commit = 0;
    cudaEvent_t ev_release = nullptr;
  };
  std::vector<Slot> st;
  long long reserved_total = 0, committed_total = 0, popped_total = 0;
  bool failed = false;                 // a commit failed after reserving its positions (traj_queue_fail)
  std::string failure;
  std::mutex mu;
  std::condition_variable cv_space, cv_ready;

  uint8_t* field(int slot, int f) { return base + (size_t)slot * slot_bytes + off[f]; }
};

namespace drl {

// Producer side.  Reserves n consecutive positions, blocking while they are not free (timeout_ms < 0: forever;
// DRL_ERR_TIMEOUT with nothing changed otherwise).  Fills `segs` with the slots they fall in; the caller enqueues its
// copies, records each segment's ev_commit on its stream, then calls traj_queue_commit.  DRL_ERR_INVALID when n
// positions can never be free at once in this queue.
int traj_queue_reserve(drl_traj_queue* q, int n, int timeout_ms, std::vector<TrajSegment>* segs);
void traj_queue_commit(drl_traj_queue* q, const std::vector<TrajSegment>& segs);
// A commit that reserved positions and then could not enqueue its copies: the positions can never be filled, so the
// queue stops instead of blocking forever.  Wakes every waiter; from then on reserve, pop and read fail with
// DRL_ERR_STATE and `why` in the message.
void traj_queue_fail(drl_traj_queue* q, const char* why);
// the largest n traj_queue_reserve can ever satisfy
int traj_queue_max_rows(const drl_traj_queue* q);

// Consumer side.  Pops the oldest full batch slot (blocking like drl_ring_pop_batch) and returns its commit events;
// traj_queue_release then records the slot's ev_release on `s` (after the caller's copies out of it) and hands it back
// to producers.
int traj_queue_pop(drl_traj_queue* q, int timeout_ms, int* slot, std::vector<cudaEvent_t>* ev_commit);
int traj_queue_release(drl_traj_queue* q, int slot, cudaStream_t s);

}  // namespace drl
