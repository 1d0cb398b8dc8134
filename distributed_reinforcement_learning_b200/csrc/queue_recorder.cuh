// queue_recorder.cuh -- the part of a policy recorder (DESIGN.md sections 12 and 13) that does not depend on the
// engine's network or on what one queue record is: the binding of one engine to one device queue for n rows, the
// device staging of n records in the queue's field order, the step word the recording kernels read, the graph that
// replays every step, the recording act's driver and the commit.  The IMPALA recorder (policy.cu: drl_policy_recorder)
// and the R2D2 recorder (r2d2_policy.cu: drl_r2d2_policy_recorder) derive from RecorderCore; each adds its kernels and
// its enqueue of one recorded step.  The A3C recorder (apex_policy.cu: drl_a3c_policy_recorder) does the same, and
// passes its commit a hook that uploads the final next_state frames.
#pragma once
#include <functional>
#include <vector>

#include "policy_core.cuh"
#include "traj_queue.cuh"

namespace drl {

struct RecorderCore {
  PolicyCore* engine = nullptr;
  QueueCore* q = nullptr;
  int n = 0, T = 0;                   // rows, steps per record
  int t = 0;                          // steps recorded since the last commit
  int f_reward = 0, f_done = 0;       // the queue fields a commit uploads from the host
  const char* last_step = "T-1";      // how the family's docs name step T-1 ("S-1" for R2D2)
  const char* commit_range = "drl:policy_recorder_commit";   // the commit's NVTX range
  uint8_t* staging = nullptr;         // [n] records, field-major in the queue's field order
  size_t off[kQueueMaxFields] = {};
  int32_t* d_t = nullptr;             // the step, read by the recording kernels
  int32_t* h_t = nullptr;             // its pinned staging
  uint8_t* h_rd = nullptr;            // pinned reward [n][T] f32 | done [n][T] u8 of a commit
  cudaGraphExec_t graph = nullptr;
  std::vector<void*> allocs;
  uint8_t* field(int f) { return staging + off[f]; }
};

// Binds r (engine, queue, n, T, f_reward, f_done set by the family) and allocates its staging, step word and pinned
// reward / done block on the engine's device.  On failure the caller releases it (recorder_core_release), keeping the
// error message.
int recorder_core_init(RecorderCore* r);
// waits for the engine's stream, frees what recorder_core_init made (the caller holds the engine's lock)
void recorder_core_release(RecorderCore* r);

template <class R>
int recorder_destroy(R* r) {
  if (!r) return DRL_OK;
  {
    std::lock_guard<std::recursive_mutex> lk(r->engine->mu);
    cudaSetDevice(r->engine->device);
    recorder_core_release(r);
  }
  delete r;
  return DRL_OK;
}

// "recorder act: all T steps ... recorded" when step T-1 is done (the caller holds the engine's lock)
int recorder_check_step(const RecorderCore* r);
// The recording act (the caller holds the engine's lock and has staged the engine's input block): the step word, then
// enqueue_step() eagerly or, with the engine's use_cuda_graph, through the recorder's graph (captured after one eager
// pass), between the engine's timing events; waits for the stream and advances the step.  The outputs are then in the
// engine's h_out.
int recorder_run_act(RecorderCore* r, const std::function<int()>& enqueue_step);
// The commit of n complete records (after step T-1; DRL_ERR_STATE otherwise): reserves n queue positions without the
// engine's lock, then, on the engine's stream, uploads reward and done into the staging, waits for each target slot's
// release event, copies every field of each segment device to device and records the segment's commit event.  A
// failure after the reservation puts the queue into its failed state (traj_queue_fail).  `before_copies`, when given,
// runs under the engine's lock after the reward / done upload and before the copies (its work goes on the engine's
// stream); its failure counts as a failure after the reservation.
int recorder_commit(RecorderCore* r, const float* reward, const uint8_t* done, int timeout_ms,
                    const std::function<int()>& before_copies = nullptr);
int recorder_reset(RecorderCore* r);

}  // namespace drl
