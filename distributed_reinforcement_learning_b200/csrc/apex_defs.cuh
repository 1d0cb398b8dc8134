// apex_defs.cuh -- definitions shared by the Ape-X / A3C learner (apex.cu), the Ape-X / A3C policy engine
// (apex_policy.cu) and the Ape-X device replay memory (apex_replay.cu): the dueling network's flat parameter layout, its
// head sizes, the learner handle and its forward + TD path.
#pragma once
#include <vector>

#include "adam_learner.cuh"
#include "kernels.h"

namespace drl {

// Offsets (in floats) inside the padded flat vectors of ONE network (FlatLayout, kernels.h).  A3C uses the same layout:
// its actor stream sits in the value* slots and its critic stream in the mean* slots (model/actor_critic.py:27-38).
struct ApexLayout : TrunkLayout {
  int64_t value1_w, value1_b, value2_w, value2_b, value3_w, value3_b;
  int64_t mean1_w, mean1_b, mean2_w, mean2_b, mean3_w, mean3_b;
  void init(int num_action) {
    A = num_action;
    const int64_t CAT = Geo::FLAT + Geo::EMB;
    const int64_t sizes[] = {
        8 * 8 * 4 * 32, 32, 4 * 4 * 32 * 64, 64, 3 * 3 * 64 * 64, 64,
        (int64_t)A * 256, 256, 256 * 256, 256,
        CAT * 256, 256, 256 * 256, 256, 256 * (int64_t)A, A,
        CAT * 256, 256, 256 * 256, 256, 256, 1};
    int64_t* const named[] = {&conv1_w, &conv1_b, &conv2_w, &conv2_b, &conv3_w, &conv3_b, &emb1_w, &emb1_b,
                              &emb2_w, &emb2_b, &value1_w, &value1_b, &value2_w, &value2_b, &value3_w, &value3_b,
                              &mean1_w, &mean1_b, &mean2_w, &mean2_b, &mean3_w, &mean3_b};
    set(sizes, named);
  }
};

constexpr int kHeadN = 2 * Geo::HID;             // 512 columns: [value hidden | mean hidden]
constexpr int kCat = Geo::FLAT + Geo::EMB;       // 3392

// drl_apex_policy_sync_from_learner: learner_params_snapshot of the main network of an Ape-X (algo 0) or A3C (algo 1)
// learner with num_action actions (DRL_ERR_INVALID for another algo or num_action)
int apex_params_snapshot(drl_apex* h, int device, int algo, int num_action, cudaStream_t dst_stream, float* dst,
                         cudaEvent_t ev_ready, cudaEvent_t ev_copied);

struct ApexActs : TrunkActs {   // forward activations of one network over up to `cap` rows (caller row order)
  float* zpart;            // [splits][M,512] split-K partial sums of the two first head layers
  float* hid1;             // [2][M,256]  value / mean stream hidden 1
  float* hid2;             // [2][M,256]
  float* vstream;          // [M,A]  value stream output
  float* scratch_sm;       // [M,A]  (softmax of the value stream: by-product of the shared output kernel, unused)
  float* mstream;          // [M]    "mean" stream output
  int cap;
};

struct ApexBwd : TrunkBwd {     // backward workspace, Mb = B rows
  float *dq, *dmean;       // [Mb,32] each (columns >= A / >= 1 stay zero)
  float *dhid2, *dhid1;    // [2][Mb,256]
};

struct ApexIn {                // views of one staging slot
  uint8_t* frames;             // [2B][84,84,4]: state rows, then next_state rows
  int32_t* pa2;                // [2B]: previous_action, then action (the embedding input of the rows s')
  float* reward;               // [B]
  uint8_t* done;               // [B]
  float* weight;               // [B]
};

}  // namespace drl

// the Ape-X / A3C learner handle (apex.cu); the device replay memory (apex_replay.cu) drives its step
struct drl_apex : drl::AdamLearner {
  drl_apex_config cfg{};
  int A = 0;
  drl::ApexLayout pl{};
  drl::ApexActs act{}, tact{};
  drl::ApexBwd bwd{};
  float *main_q = nullptr, *next_main_q = nullptr, *target_q = nullptr, *target_value = nullptr, *sav = nullptr,
        *td_dev = nullptr;
  // A3C runs on the same body (drl_a3c_*): no target scope, the A3C loss kernel of apex.cu, three loss scalars
  int algo = 0;                // 0 = Ape-X DQN, 1 = A3C
  float a3c_baseline_coef = 0.f, a3c_entropy_coef = 0.f;
  int a3c_clip = 0;
  float* adv = nullptr;        // [B] advantage tap
  std::vector<drl::ApexIn> in;      // per slot
};

namespace drl {

// forward passes + TD kernel over n transitions held by `sl` on the compute stream (the target forward on its own stream
// pair when the step runs parallel); train = also the head gradients and the loss.  Writes |target - q(s, a)| to td_dev
// and, when td_host is not null, to td_host.  Adds the launches to *launches unless it is null.
int enqueue_forward_td(drl_apex* h, const ApexIn& sl, int n, bool train, float* td_host, int* launches);

}  // namespace drl
