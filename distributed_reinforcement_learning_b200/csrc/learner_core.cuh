// learner_core.cuh -- the learner-handle core of every learner handle: the IMPALA handle (learner.cu) and, through the
// Adam layer (adam_learner.cuh), the Ape-X / A3C (apex.cu) and R2D2 (r2d2.cu) handles (DESIGN.md section 6).  It knows
// neither the network nor the optimizer: streams, parameters, the gradient bucket, staging slots, result rows, the step
// graphs, and the C-ABI bodies that are the same in every family.  A family derives its handle from LearnerCore and
// plugs in two hooks: fwd_bwd (forward + loss + backward of a staged slot) and update (the optimizer).
#pragma once
#include <mutex>
#include <vector>

#include "kernels.h"

namespace drl {

struct LearnerSlot {
  uint8_t* base = nullptr;          // one allocation; the family's views of its fields point into it
  cudaEvent_t staged = nullptr;     // H2D of this slot finished (copy stream)
  cudaEvent_t consumed = nullptr;   // last compute that read this slot finished (compute stream)
  bool has_data = false;
};

struct LearnerCore {
  // Enqueues forward, loss and backward of the batch staged in `slot` on the compute stream, leaving the gradients and
  // the loss sums in the bucket; adds its kernel launches to *launches unless it is null.
  using FwdBwd = int (*)(LearnerCore* h, int slot, int* launches);
  // Enqueues the optimizer update (two kernels) on the compute stream; it writes the step's 8 scalars into result row
  // out_row.  grad_scale multiplies the bucket (data parallel); local_only: update from the local bucket even when the
  // family reduces it across replicas itself; early: the backward pass of the same enqueue ran just before.
  using Update = int (*)(LearnerCore* h, int out_row, float grad_scale, bool local_only, bool early);

  // One handle is used by one host thread at a time, but actor threads call parameter_sync -> get_params / the
  // snapshot on the learner's handle while the learner thread trains, and ctypes drops the GIL: every C-ABI entry point
  // takes this lock (h_flat, `pending`, the result rows and the graph caches are all guarded by it).
  mutable std::recursive_mutex mu;
  // set by the family before learner_core_init
  int device = 0, num_slots = 2, B = 0, mode = 2;
  int scratch_slots = 0;                   // staging slots past num_slots for the family's synchronous calls
  bool use_cuda_graph = false;
  const TrunkLayout* layout = nullptr;     // the family's network
  FwdBwd fwd_bwd = nullptr;
  Update update = nullptr;

  cudaStream_t compute = nullptr, copy = nullptr, side = nullptr;
  cudaEvent_t fj[8] = {};                  // fork/join events between the compute and the side stream
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  bool par = true;                         // run off-critical-path kernels on the side stream
  bool images_stale = true;                // the main weight images do not match the parameters
  float* params = nullptr;
  float* grads = nullptr;                  // the bucket [padded_total grads | 4 loss sums]: one all-reduce covers both
  float* loss = nullptr;                   // = grads + padded_total
  long long* d_step = nullptr;
  float* d_lr = nullptr;
  // mapped pinned [num_slots + 1][8]: the steps' scalars, written by the update kernel itself (zero-copy).  Row = slot
  // for a step, row num_slots for the data-parallel apply, so that two steps on two slots can be in flight.
  float *h_out = nullptr, *d_out = nullptr;
  std::vector<cudaEvent_t> ev_done;        // per result row
  float* h_flat = nullptr;                 // pinned staging of set/get params (padded_total floats)
  std::vector<LearnerSlot> slots;          // num_slots training slots + scratch_slots
  std::vector<void*> allocs;
  std::vector<cudaGraphExec_t> graph_step, graph_fb;   // per slot: the whole step; the forward_backward half
  cudaGraphExec_t graph_apply = nullptr;   // the apply half, captured with grad_scale graph_apply_scale
  float graph_apply_scale = 0.f;
  bool pending = false;                    // a step was enqueued and its scalars not yet collected
  int last_row = 0;                        // result row of the most recently enqueued update
  int last_slot = 0;                       // slot of the most recent step / forward_backward
  int last_n = 0;                          // rows of the most recent training or forward-only pass (taps, read_buffer)
  int launches = 0;                        // kernel launches of one step (valid after the first step)

  Streams streams() const;
};

// Streams, events, parameters, the bucket, pinned buffers and num_slots + scratch_slots staging slots of slot_bytes
// each.  On failure the caller destroys the handle (learner_core_release).
int learner_core_init(LearnerCore* h, size_t slot_bytes);
void learner_core_release(LearnerCore* h);   // frees everything learner_core_init and dev_alloc made

int set_device(const LearnerCore* h);
// `family` names the handle type in the null-handle message ("null <family> handle")
int check_handle(const LearnerCore* h, const char* family);
int check_slot(const LearnerCore* h, int slot);
// packed host vector <-> padded device vector of the layout, through h_flat on the compute stream; upload fills the
// padding with pad_value (the caller has checked the length and set the device)
int learner_upload(LearnerCore* h, float* dev_padded, const float* host_packed, float pad_value);
int learner_download(LearnerCore* h, const float* dev_padded, float* host_packed);

// C-ABI bodies
int learner_param_count(const LearnerCore* h, const char* family, int64_t* n);
int learner_set_params(LearnerCore* h, const char* family, const float* host_flat, int64_t n);
int learner_get_params(LearnerCore* h, const char* family, float* host_flat, int64_t n);
// `bucket`: the padded gradient vector to read (the local bucket, or the family's reduced copy of it)
int learner_get_grads(LearnerCore* h, const char* family, const float* bucket, float* host_flat, int64_t n);
int learner_grad_bucket(LearnerCore* h, const char* family, void** dev_ptr, int64_t* count);
// Parameter snapshot for a policy engine, under the learner's lock: records ev_ready on the compute stream (after
// everything enqueued so far, a step in flight included), makes dst_stream wait for it, copies the padded main
// parameters device to device into dst on dst_stream, records ev_copied there and makes the compute stream wait for it,
// so that the next update cannot overwrite the parameters while they are read.  Does not block the host.
// DRL_ERR_INVALID for a learner on another device; the family checks that the networks match.
int learner_params_snapshot(LearnerCore* h, const char* family, int device, cudaStream_t dst_stream, float* dst,
                            cudaEvent_t ev_ready, cudaEvent_t ev_copied);
int learner_step_async(LearnerCore* h, const char* family, int slot);
// the body of learner_step_async (the caller holds the lock and has set the device): waits for the slot's `staged`
// event, enqueues forward + loss + backward + update into result row `slot` (graph or eager) on the compute stream,
// records `consumed`, ev_stop and the row's done event, marks the step pending
int learner_run_step(LearnerCore* h, int slot);
// data parallel: the step in two halves around the caller's reduction of the bucket (graphs under use_cuda_graph)
int learner_forward_backward(LearnerCore* h, const char* family, int slot);
int learner_apply(LearnerCore* h, const char* family, float grad_scale);
// wait for the step in flight / for the last step on `slot`; *row = its 8 scalars
int learner_wait(LearnerCore* h, const char* family, const float** row);
int learner_wait_slot(LearnerCore* h, const char* family, int slot, const float** row);
// one step with par = false and a CUDA event before every named launch
int learner_profile_step(LearnerCore* h, const char* family, int slot, char* names, int64_t names_len, float* ms,
                         int32_t max_kernels, int32_t* count);
int learner_last_step_ms(LearnerCore* h, const char* family, float* ms);
int learner_stream(LearnerCore* h, const char* family, void** stream);
int learner_launches_per_step(const LearnerCore* h, const char* family, int32_t* n);

int64_t step_of(const float* row);              // global_step from the two words at row[6], row[7]

struct NamedBuffer { const char* name; const float* p; size_t count; };
// copies the buffer called `name` out of tab[0, ntab) (after the compute stream drains)
int read_named_buffer(LearnerCore* h, const NamedBuffer* tab, int ntab, const char* name, float* host_dst, int64_t n);

}  // namespace drl
