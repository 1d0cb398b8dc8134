// replay_core.cuh -- the part of a device prioritized replay memory that does not depend on what one record is
// (DESIGN.md sections 10 and 11): the float64 sum tree of buffer_queue.SumTree (distributed_queue/buffer_queue.py:326-371)
// on the device with its two kernels (replay_core.cu), the host state that follows from the call sequence (write cursor,
// n_entries, beta), the last sample's device buffers, the pinned blocks of the host -> device traffic, the event that
// orders the memory's work, and the C-ABI bodies of sample / update / last_sample / total / size / beta.
//
// A family (apex_replay.cu: one transition per record; r2d2_replay.cu: one sequence per record) derives its handle from
// ReplayCore, adds its record storage and its store / gather kernels, and drives a learner's step through replay_step.
// All work of a memory is totally ordered: each call makes the stream it enqueues on wait for `ev_last` (replay_begin:
// recorded after the previous call's last enqueue, on whichever stream that was) and records it again after its own
// last enqueue (replay_end).
#pragma once
#include <functional>
#include <mutex>
#include <vector>

#include "adam_learner.cuh"
#include "kernels.h"

namespace drl {

constexpr double kReplayE = 0.001, kReplayA = 0.6, kReplayBetaInc = 0.001;   // Memory.e / a / beta increment (:373-376)
// One warp per tree level in the update kernel: depth(2 * capacity - 2) <= 32 levels below the root.
constexpr int64_t kReplayMaxCapacity = int64_t(1) << 31;

// one pinned, device-mapped host block reused call after call; `ev` is recorded after the last device work that reads
// it, and the host waits for it before writing the block again
struct PinnedBlock {
  uint8_t* h = nullptr;
  uint8_t* d = nullptr;           // device alias of h
  size_t bytes = 0;
  cudaEvent_t ev = nullptr;
};

struct ReplayCore {
  const char* family = "replay";       // names the memory in error messages ("null <family> handle", "<family> sample: ...")
  int device = 0;
  int64_t capacity = 0;
  int levels = 0;                      // warps of the tree update kernel
  cudaStream_t stream = nullptr;       // calls that use no learner
  cudaEvent_t ev_last = nullptr;       // after the memory's last enqueue
  double* tree = nullptr;              // [2 * capacity - 1]
  // the last sample, on the device
  int64_t *d_tree_index = nullptr, *d_data_index = nullptr;
  double *d_priority = nullptr, *d_is_weight = nullptr;
  int sample_cap = 0, last_n = 0;
  // ingest: pinned block -> one H2D -> the device block (the family's layout, ingest_bytes of room)
  PinnedBlock ingest;
  uint8_t* d_ingest = nullptr;
  size_t ingest_bytes = 0;
  PinnedBlock args;                    // the uniforms / indices / errors of calls without a learner
  std::vector<PinnedBlock> uniforms;   // per learner slot: the uniforms of replay_step
  // host-side state of Memory that follows from the call sequence (per.cu keeps the same, in the same types)
  int64_t cursor = 0, n_entries = 0;
  double beta = 0.4;
  std::vector<void*> allocs;           // the family's record storage and the tree (dev_alloc)
  std::recursive_mutex mu;
};

// "null <family> handle" for a null r
int replay_check(const ReplayCore* r, const char* family);
// capacity in [2, 2^31] and a device to run on (checked in that order; the family checks its own arguments first)
int replay_check_create(const char* family, int32_t device, int64_t capacity);
// stream, ev_last and the zero-initialised tree; on failure the caller releases the handle (replay_core_release)
int replay_core_init(ReplayCore* r, int device, int64_t capacity);
// waits for the memory's work, frees everything replay_core_init, dev_alloc and the pinned blocks made
void replay_core_release(ReplayCore* r);

// waits until the device no longer reads the block, growing it to `bytes` first if needed
int replay_acquire(PinnedBlock& b, size_t bytes);
// the ingest blocks (pinned and device) with room for `bytes`; regrowing the device block waits for earlier work
int replay_ensure_ingest(ReplayCore* r, size_t bytes);
// the last-sample buffers with room for n draws
int replay_ensure_sample(ReplayCore* r, int n);
// the stream of this call, ordered after the memory's previous work / record ev_last after this call's last enqueue
int replay_begin(ReplayCore* r, cudaStream_t s);
int replay_end(ReplayCore* r, cudaStream_t s);
// Memory.add / Memory.update of n leaves in order: tree_index[i], or the leaves at the write cursor `first` onwards when
// tree_index is null; errors err64 (double) or, when it is null, err32 (float, a learner's |td|)
int replay_launch_update(ReplayCore* r, cudaStream_t s, int n, const int64_t* tree_index, int64_t first,
                         const double* err64, const float* err32);
// Memory.sample's beta step (:395) and the sample kernel over n draws with the uniforms at u01_dev; the importance
// weights also go to weight32 as float32 when it is not null
int replay_launch_sample(ReplayCore* r, cudaStream_t s, int n, const double* u01_dev, float* weight32);
int replay_check_u01(const ReplayCore* r, int n, const double* u01);
// SumTree.add's cursor and n_entries after n records were stored at the cursor (:351-359)
void replay_advance(ReplayCore* r, int n);

// The training half of one learner-loop iteration on the learner's compute stream (the caller holds both locks and has
// checked the learner and the slot): Memory.sample(B) with the uniforms u01 [B], the importance weights as float32 into
// `weight32` (the slot's weight view), gather(stream) of the sampled rows r->d_data_index [B] into the slot (after an
// earlier drl_*_stage of the slot), the learner's step (learner_run_step), and Memory.update of the sampled leaves with
// the step's |td| (td_dev), before the done event of the learner's result row.  DRL_ERR_STATE on an empty memory.
int replay_step(ReplayCore* r, AdamLearner* learner, int slot, const double* u01, float* weight32, const float* td_dev,
                const std::function<int(cudaStream_t)>& gather);

// C-ABI bodies (the family passes its handle and its name for the null-handle message)
int replay_sample(ReplayCore* r, const char* family, int32_t n, const double* u01, int64_t* tree_index,
                  int64_t* data_index, double* priority, double* is_weight);
int replay_update(ReplayCore* r, const char* family, int32_t n, const int64_t* tree_index, const double* error);
int replay_last_sample(ReplayCore* r, const char* family, int64_t* tree_index, double* priority, double* is_weight);
int replay_total(ReplayCore* r, const char* family, double* total);
int replay_size(ReplayCore* r, const char* family, int64_t* n_entries);
int replay_beta(ReplayCore* r, const char* family, double* beta);

}  // namespace drl
