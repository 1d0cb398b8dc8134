// policy_core.cuh -- the part of a batched policy engine that does not depend on the network (DESIGN.md section 7):
// the engine's stream and events, its parameters, the conv weight images and the action-embedding table derived from
// them, the conv activations and split-K partials of up to max_batch rows, the pinned input block and the mapped output
// block, one graph per row count, and the C-ABI bodies that are the same for every engine.
//
// A family (policy.cu: IMPALA; r2d2_policy.cu: R2D2; apex_policy.cu: Ape-X and A3C) derives its handle from
// PolicyCore, checks its config, lays out its input and output blocks, and passes its act through one hook
// (enqueue_act).  Its act entry point checks its arguments, stages its inputs into h_in, runs policy_run_act and copies
// its outputs out of h_out.
#pragma once
#include <functional>
#include <mutex>
#include <vector>

#include "kernels.h"

namespace drl {

struct PolicyCore {
  // Enqueues the act of n rows on the engine's stream: one H2D of the staged input block, then the family's kernels,
  // which write their outputs to mapped memory (d_out).
  using EnqueueAct = int (*)(PolicyCore* h, int n);
  // The conv2 / conv3 forward weight images of the parameters (conv_images16 or conv_images_tf32).
  using ConvImages = int (*)(cudaStream_t s, const TrunkLayout& pl, const float* params, uint8_t* img_conv2,
                             uint8_t* img_conv3);

  // every C-ABI entry point but param_count locks the handle (actor threads share an engine; ctypes drops the GIL)
  std::recursive_mutex mu;
  // set by the family before policy_core_init
  int device = 0, max_batch = 0, A = 0;
  int splits = 0, zpart_cols = 0;         // zpart is [splits][n][zpart_cols] for an act of n rows
  bool use_cuda_graph = false;
  const TrunkLayout* layout = nullptr;    // the family's layout (the learner's)
  EnqueueAct enqueue_act = nullptr;
  ConvImages conv_images = nullptr;

  cudaStream_t stream = nullptr;
  cudaEvent_t ev_ready = nullptr, ev_copied = nullptr;   // learner -> policy and policy -> learner edges of a sync
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;     // device time of the last act
  bool timed = false;
  int last_n = 0;                // rows of the most recent act or recorder act (0: none yet), for policy_read_buffer
  float* params = nullptr;       // padded flat vector (learner layout)
  uint8_t* img_conv2 = nullptr;  // conv2 / conv3 forward weight images
  uint8_t* img_conv3 = nullptr;
  float* e1 = nullptr;           // [A,256] relu(emb1), scratch of emb_forward
  float* table = nullptr;        // [A,256] action-embedding table (depends on the parameters only)
  float *a1 = nullptr, *a2 = nullptr, *a3 = nullptr;   // conv activations of max_batch rows
  uint16_t *a1p = nullptr, *a2p = nullptr;              // 16-bit planes of a1 / a2 (conv_forward16)
  float* zpart = nullptr;        // split-K partial sums of the family's first skinny GEMM
  uint8_t* d_in = nullptr;       // device input block (the family's layout)
  uint8_t* h_in = nullptr;       // pinned staging of the same block
  uint8_t* h_out = nullptr;      // mapped pinned outputs (the family's layout)
  uint8_t* d_out = nullptr;      // its device alias
  std::vector<cudaGraphExec_t> graphs;   // per row count n
  std::vector<void*> allocs;
};

// create's device check ("no CPU fallback"), after the family has checked its config
int policy_check_device(int device);
// Sets the device and the family's kernel attributes (set_attributes), then makes the stream, the events, the
// parameters, the weight images, the table, the conv activations, zpart_floats of split-K partials, the input block of
// in_bytes (device + pinned) and the mapped output block of out_bytes, and derives the table and the images of the zero
// parameters.  On failure it releases what it made, keeping the error message, and the family deletes the handle.
int policy_core_init(PolicyCore* h, int (*set_attributes)(), size_t zpart_floats, size_t in_bytes, size_t out_bytes);
// waits for the engine's stream, frees everything policy_core_init and dev_alloc made
void policy_core_release(PolicyCore* h);

template <class H>
int policy_destroy(H* h) {
  if (!h) return DRL_OK;
  policy_core_release(h);
  delete h;
  return DRL_OK;
}

// The act driver (the caller holds the lock and has staged n rows into h_in): ev_start, then the family's enqueue_act
// eagerly or, with use_cuda_graph, through the graph of n (captured after one eager pass: the launchers set their
// kernel attributes and build their tensor maps outside capture), ev_stop, and a wait for the stream; the outputs are
// then in h_out.
int policy_run_act(PolicyCore* h, int n);
// act's checks shared by the families: n in [1, max_batch], and no null input (inputs_given)
int policy_check_n(const PolicyCore* h, int n, bool inputs_given);
// row by row: previous_action[i] in [0, A) unless previous_action is null, explore[i] in [-1, A) unless explore is null
int policy_check_actions(const PolicyCore* h, int n, const int32_t* previous_action, const int32_t* explore);
// the explore actions of n rows into the staging block, or -1 ("greedy") for every row when explore is null
void policy_stage_explore(uint8_t* dst, const int32_t* explore, int n);

// C-ABI bodies.  `family` names the engine in the null-handle message ("null <family> handle") and, with its spaces as
// underscores, in the NVTX ranges ("drl:r2d2_policy_sync").
int policy_check(const PolicyCore* h, const char* family);
int policy_param_count(const PolicyCore* h, const char* family, int64_t* n);
int policy_set_params(PolicyCore* h, const char* family, const float* host_flat, int64_t n);
int policy_get_params(PolicyCore* h, const char* family, float* host_flat, int64_t n);
// parameter_sync: `snapshot` is the family's learner snapshot (impala_params_snapshot, r2d2_params_snapshot or
// apex_params_snapshot) of `learner` into params on the engine's stream, ordered by ev_ready / ev_copied
int policy_sync(PolicyCore* h, const char* family, const void* learner, const std::function<int()>& snapshot);
int policy_last_act_ms(PolicyCore* h, const char* family, float* ms);
// Test aid: a copy of one buffer of the most recent act (policy_run_act or recorder_run_act, last_n rows) into host
// memory, after the engine's stream: "a1" [n,20,20,32], "a2" [n,9,9,64], "a3" [n,3136], "e1" / "table" [A,256],
// "zpart" [splits][n][zpart_cols].  n = element count (DRL_ERR_INVALID if it differs, or for an unknown name);
// DRL_ERR_STATE before the first act.  A policy server's serve does not go through the act driver: it neither sets
// last_n nor keeps these buffers as the last act left them.
int policy_read_buffer(PolicyCore* h, const char* family, const char* name, float* host_dst, int64_t n);
// out[0] = last_n (0 before the first act), out[1] = splits, out[2] = zpart_cols
int policy_buffer_dims(PolicyCore* h, const char* family, int32_t* out);

}  // namespace drl
