// r2d2_defs.cuh -- definitions shared by the R2D2 learner (r2d2.cu), the R2D2 policy engine (r2d2_policy.cu) and the
// R2D2 device replay memory (r2d2_replay.cu): the network's sizes, its flat parameter layout, the learner handle and its
// forward + TD path.
#pragma once
#include <vector>

#include "adam_learner.cuh"
#include "kernels.h"

namespace drl {

// lstm_size of config.json:93: the width of the policy engine, recorder and device queue, and the learner width whose
// recurrence runs one CTA per sequence (r2d2_lstm_fwd_kernel); the learner also takes 256 and 512 (r2d2_cluster.cuh)
constexpr int kR2L = 64;
constexpr int kR2G = 4 * kR2L;           // 256 gate columns
constexpr int kR2H = 128;                // dense width between the LSTM and the two output streams (model/r2d2_lstm.py:50)
constexpr int kR2Cat = Geo::FLAT + Geo::EMB;   // 3392 rows of the LSTM kernel that multiply the step input

struct R2Layout : TrunkLayout {
  int64_t lstm_w, lstm_b, q1_w, q1_b, value_w, value_b, mean_w, mean_b;
  void init(int num_action, int channels, int L = kR2L) {
    A = num_action; C = channels;
    const int64_t sizes[] = {
        8 * 8 * (int64_t)C * 32, 32, 4 * 4 * 32 * 64, 64, 3 * 3 * 64 * 64, 64,
        (int64_t)A * 256, 256, 256 * 256, 256,
        (int64_t)(kR2Cat + L) * 4 * L, 4 * L,
        (int64_t)L * kR2H, kR2H, (int64_t)kR2H * A, A, kR2H, 1};
    int64_t* const named[] = {&conv1_w, &conv1_b, &conv2_w, &conv2_b, &conv3_w, &conv3_b, &emb1_w, &emb1_b, &emb2_w,
                              &emb2_b, &lstm_w, &lstm_b, &q1_w, &q1_b, &value_w, &value_b, &mean_w, &mean_b};
    set(sizes, named);
  }
};

// drl_r2d2_policy_sync_from_learner: learner_params_snapshot of an R2D2 learner whose network has num_action actions,
// `channels` input channels and lstm_size kR2L, the policy engine's (DRL_ERR_INVALID otherwise)
int r2d2_params_snapshot(drl_r2d2* h, int device, int num_action, int channels, cudaStream_t dst_stream, float* dst,
                         cudaEvent_t ev_ready, cudaEvent_t ev_copied);

struct R2Acts : TrunkActs {   // activations of one scope, time-major rows m = t*B + b
  float* zpart;            // [splits][M, 4L]: [a3 | emb] W_x partial sums
  float* zx;               // [M, 4L]: their sum (the recurrence reads one value per gate and step)
  float* gates;            // [M, 4L] sigmoid(i), tanh(j), sigmoid(f + 1), sigmoid(o)
  float *tc, *hout;        // [M, L] tanh(c_t), h_t (the cell output, BEFORE the done mask)
  float *hin, *cin;        // [M, L] the (masked) state that entered step t
  float* q1;               // [M, 128]
  float* q;                // [M, A]
};
struct R2Bwd : TrunkBwd {     // backward workspace, all M rows
  float *dq, *dmean;       // [M, 32]
  float *dq1, *dhout, *dz; // [M,128], [M,L], [M,4L]
};
struct R2In {              // one staged minibatch, caller's batch-major layout
  const uint8_t* frames;   // [B, S, 84, 84, C]
  const int32_t* pa;       // [B, S]
  const int32_t* action;   // [B, S]
  const float* h0;         // [B, L]
  const float* c0;         // [B, L]
  const float* reward;     // [B, S]
  const uint8_t* done;     // [B, S]
  const float* weight;     // [B]
};

}  // namespace drl

// the R2D2 learner handle (r2d2.cu); the device replay memory (r2d2_replay.cu) drives its step
struct drl_r2d2 : drl::AdamLearner {
  drl_r2d2_config cfg{};
  int S = 0, A = 0, C = 1, Nt = 0;
  int L = drl::kR2L;                    // lstm_size: 64, 256 or 512
  int clusters_fwd = 0, clusters_bwd = 0;   // L > 64: clusters of the recurrence kernels the device places at once
  size_t frame = 0;
  drl::R2Layout pl{};
  drl::R2Acts act{}, tact{};
  drl::R2Bwd bwd{};
  float *sav = nullptr, *target_value = nullptr, *td_dev = nullptr, *c_last = nullptr;
  std::vector<drl::R2In> in;            // per slot
};

namespace drl {

// both unrolls (main and target scope) + TD kernel over the nb sequences held by `in` on the compute stream (the target
// unroll on its own stream pair when the step runs parallel); train = also the head gradients and the loss.  Writes
// the per-sequence priority (|mean_t(target - q)|, or the mixed max / mean rule of cfg.priority_rule) to td_dev and, when
// td_host is not null, to td_host.  Adds the launches to *launches unless it is null.
int enqueue_forward_td(drl_r2d2* h, const R2In& in, int nb, bool train, float* td_host, int* launches);

}  // namespace drl
