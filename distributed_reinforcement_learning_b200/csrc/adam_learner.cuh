// adam_learner.cuh -- the learner-handle core shared by the Ape-X / A3C handle (apex.cu) and the R2D2 handle (r2d2.cu):
// streams, main and target parameters, TF1 Adam state, staging slots, the per-slot step graph, and the C-ABI bodies
// that do not depend on the network (DESIGN.md section 6).  A family derives its handle from AdamLearner, adds its
// activations and slot views, and passes its forward + loss + backward through one hook (fwd_bwd).
#pragma once
#include <mutex>
#include <vector>

#include "kernels.h"

namespace drl {

struct AdamSlot {
  uint8_t* base = nullptr;          // one allocation; the family's views of its fields point into it
  cudaEvent_t staged = nullptr;     // H2D of this slot finished (copy stream)
  cudaEvent_t consumed = nullptr;   // last compute that read this slot finished (compute stream)
  bool has_data = false;
};

struct AdamLearner {
  // Enqueues forward, TD / policy loss and backward of the minibatch staged in `slot` on the compute stream (the Adam
  // update follows it); adds the kernel launches to *launches unless it is null.
  using FwdBwd = int (*)(AdamLearner* h, int slot, int* launches);

  // every C-ABI entry point locks the handle (actor threads call parameter_sync -> get_params on the learner's handle
  // while the learner thread trains; ctypes drops the GIL)
  mutable std::recursive_mutex mu;
  // set by the family before adam_learner_init
  int device = 0, num_slots = 2, B = 0, mode = 2;
  bool use_cuda_graph = false;
  const TrunkLayout* layout = nullptr;     // the family's layout (one network)
  FwdBwd fwd_bwd = nullptr;

  cudaStream_t compute = nullptr, copy = nullptr, side = nullptr;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr, ev_done = nullptr;
  cudaEvent_t fj[8] = {};
  // the target scope's forward is independent of the main scope's: it runs on its own stream pair beside it
  cudaStream_t tmain = nullptr, tside = nullptr;
  cudaEvent_t tfj[8] = {}, ev_tfork = nullptr, ev_tjoin = nullptr;
  bool par = true;
  float *params = nullptr, *target = nullptr, *adam_m = nullptr, *adam_v = nullptr;
  float* grads = nullptr;                  // [padded_total grads | 4 loss scalars]: one all-reduce covers both
  float* loss = nullptr;                   // = grads + padded_total
  WeightImages wi{}, twi{};
  bool main_images_stale = true, target_images_stale = true;
  AdamState opt{};                         // the family sets start_lr, end_lr, learning_frame and clip_norm
  long long* d_step = nullptr;
  float *d_lr = nullptr, *d_alpha = nullptr, *d_b1p = nullptr, *d_b2p = nullptr;
  float *h_out = nullptr, *d_out = nullptr;   // mapped pinned [num_slots][8]: the step scalars
  float *h_td = nullptr, *d_td = nullptr;     // mapped pinned [num_slots][B]: the new priorities
  float* h_flat = nullptr;                    // pinned staging of set/get params (padded_total floats)
  float* h_ones = nullptr;                    // pinned 1.0f: the importance weights staged when the caller passes none
  std::vector<AdamSlot> slots;                // num_slots training slots + 1 scratch slot for the synchronous calls
  std::vector<void*> allocs;
  std::vector<cudaGraphExec_t> graph_step;
  bool pending = false;
  int last_slot = 0;
  int last_n = 0;                             // minibatch of the most recent step / td_error call (taps, read_buffer)
  int launches = 0;

  Streams streams() const;
  Streams target_streams() const;   // own pair when the step runs parallel, otherwise the main pair (serial)
};

// Streams, events, parameters, Adam state, pinned buffers and num_slots + 1 staging slots of slot_bytes each; `ones`
// unit weights.  On failure the caller destroys the handle (adam_learner_release).
int adam_learner_init(AdamLearner* h, size_t slot_bytes, size_t ones);
void adam_learner_release(AdamLearner* h);      // frees everything adam_learner_init and dev_alloc made
int adam_step(cudaStream_t s, const AdamState& o);

// C-ABI bodies.  `family` names the handle type in the null-handle message ("null <family> handle").
int check_handle(const AdamLearner* h, const char* family);
int check_slot(const AdamLearner* h, int slot);
int adam_param_count(const AdamLearner* h, const char* family, int64_t* n);
int adam_set_params(AdamLearner* h, const char* family, int which, const float* host_flat, int64_t n);
int adam_get_params(AdamLearner* h, const char* family, int which, float* host_flat, int64_t n);
int adam_set_opt_state(AdamLearner* h, const char* family, const float* host_m, const float* host_v, int64_t n,
                       int64_t step, float beta1_power, float beta2_power);
int adam_get_opt_state(AdamLearner* h, const char* family, float* host_m, float* host_v, int64_t n, int64_t* step,
                       float* beta1_power, float* beta2_power);
int adam_get_grads(AdamLearner* h, const char* family, float* host_flat, int64_t n);
int adam_main_to_target(AdamLearner* h, const char* family);
// Parameter snapshot for a policy engine, under the learner's lock: records ev_ready on the compute stream (after
// everything enqueued so far, a step in flight included), makes dst_stream wait for it, copies the padded main
// parameters device to device into dst on dst_stream, records ev_copied there and makes the compute stream wait for it,
// so that the next update cannot overwrite the parameters while they are read.  Does not block the host.
// DRL_ERR_INVALID for a learner on another device; the family checks that the networks match.
int adam_params_snapshot(AdamLearner* h, const char* family, int device, cudaStream_t dst_stream, float* dst,
                         cudaEvent_t ev_ready, cudaEvent_t ev_copied);
int adam_step_async(AdamLearner* h, const char* family, int slot);
// the body of adam_step_async (the caller holds the lock and has set the device): waits for the slot's `staged` event,
// enqueues forward + loss + backward + update (graph or eager) on the compute stream, records `consumed`, ev_stop and
// ev_done, marks the step pending
int adam_run_step(AdamLearner* h, int slot);
int adam_forward_backward(AdamLearner* h, const char* family, int slot);
int adam_grad_bucket(AdamLearner* h, const char* family, void** dev_ptr, int64_t* count);
int adam_apply(AdamLearner* h, const char* family, float grad_scale);
// waits for the step in flight; *row = its 8 scalars (adam_apply_kernel), td_error = its B priorities (may be null)
int adam_wait(AdamLearner* h, const char* family, const float** row, float* td_error);
int adam_profile_step(AdamLearner* h, const char* family, int slot, char* names, int64_t names_len, float* ms,
                      int32_t max_kernels, int32_t* count);
int adam_last_step_ms(AdamLearner* h, const char* family, float* ms);
int adam_stream(AdamLearner* h, const char* family, void** stream);
int adam_launches_per_step(const AdamLearner* h, const char* family, int32_t* n);

int64_t step_of(const float* row);              // global_step from the two words at row[6], row[7]

struct NamedBuffer { const char* name; const float* p; size_t count; };
// copies the buffer called `name` out of tab[0, ntab) (after the compute stream drains)
int read_named_buffer(AdamLearner* h, const NamedBuffer* tab, int ntab, const char* name, float* host_dst, int64_t n);

}  // namespace drl
