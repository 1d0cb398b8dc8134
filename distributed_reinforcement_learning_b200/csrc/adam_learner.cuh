// adam_learner.cuh -- the Adam layer of the Ape-X / A3C handle (apex.cu) and the R2D2 handle (r2d2.cu) on the
// learner-handle core (learner_core.cuh, DESIGN.md section 6): the target network, TF1 Adam state and the new priorities.
// A family derives its handle from AdamLearner, adds its activations and slot views, and passes its forward + loss +
// backward through the core's fwd_bwd hook; the update hook is Adam's.
#pragma once
#include "learner_core.cuh"

namespace drl {

struct AdamLearner : LearnerCore {
  // the target scope's forward is independent of the main scope's: it runs on its own stream pair beside it
  cudaStream_t tmain = nullptr, tside = nullptr;
  cudaEvent_t tfj[8] = {}, ev_tfork = nullptr, ev_tjoin = nullptr;
  float *target = nullptr, *adam_m = nullptr, *adam_v = nullptr;
  WeightImages wi{}, twi{};
  bool target_images_stale = true;
  AdamState opt{};                         // the family sets start_lr, end_lr, learning_frame and clip_norm
  float *d_alpha = nullptr, *d_b1p = nullptr, *d_b2p = nullptr;
  float *h_td = nullptr, *d_td = nullptr;     // mapped pinned [num_slots][B]: the new priorities
  float* h_ones = nullptr;                    // pinned 1.0f: the importance weights staged when the caller passes none

  Streams target_streams() const;   // own pair when the step runs parallel, otherwise the main pair (serial)
};

// The core (one scratch slot for the synchronous calls), the target stream pair, target parameters, Adam state and
// `ones` unit weights.  On failure the caller destroys the handle (adam_learner_release).
int adam_learner_init(AdamLearner* h, size_t slot_bytes, size_t ones);
void adam_learner_release(AdamLearner* h);      // frees everything adam_learner_init and dev_alloc made
int adam_step(cudaStream_t s, const AdamState& o);

// C-ABI bodies.  `family` names the handle type in the null-handle message ("null <family> handle").
int adam_set_params(AdamLearner* h, const char* family, int which, const float* host_flat, int64_t n);
int adam_get_params(AdamLearner* h, const char* family, int which, float* host_flat, int64_t n);
int adam_set_opt_state(AdamLearner* h, const char* family, const float* host_m, const float* host_v, int64_t n,
                       int64_t step, float beta1_power, float beta2_power);
int adam_get_opt_state(AdamLearner* h, const char* family, float* host_m, float* host_v, int64_t n, int64_t* step,
                       float* beta1_power, float* beta2_power);
int adam_main_to_target(AdamLearner* h, const char* family);
// waits for the step in flight; *row = its 8 scalars (adam_apply_kernel), td_error = its B priorities (may be null)
int adam_wait(AdamLearner* h, const char* family, const float** row, float* td_error);

}  // namespace drl
