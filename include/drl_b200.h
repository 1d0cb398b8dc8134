/*
 * drl_b200.h -- C-ABI of the H100-native learner hot paths: IMPALA (the headline path), then the Ape-X DQN, R2D2 and
 * A3C learner steps and the prioritized-replay index (SURVEY.md section 8(f)).
 *
 * The reference (chagmgang/distributed_reinforcement_learning @ 1890ce4) has no FFI: its hot
 * path is a Python call surface over a TF1 graph.  This header is what a replacement of that
 * path binds (ctypes today; see INTEGRATION.md).  Every entry point names the reference
 * interface it replaces (file:line under /root/reference).
 *
 * Conventions: extern "C"; plain pointers and sizes; every function returns int
 * (0 = ok, <0 = error, text via drl_last_error()); no exception crosses the boundary;
 * pointers are caller-owned unless produced by a *_create; a handle is used by one host
 * thread at a time (the ring is the exception: it is multi-producer / single-consumer safe).
 * "host" pointers are CPU memory (pinned or pageable), "dev" pointers are CUDA device memory.
 * There is NO CPU fallback: without a CUDA device every compute entry point fails with
 * DRL_ERR_CUDA.
 */
#ifndef DRL_B200_H_
#define DRL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DRL_OK 0
#define DRL_ERR_INVALID (-1) /* bad argument / unsupported configuration */
#define DRL_ERR_CUDA (-2)    /* CUDA runtime error (text in drl_last_error) */
#define DRL_ERR_STATE (-3)   /* call out of order (e.g. step before stage) */
#define DRL_ERR_TIMEOUT (-4) /* ring wait timed out */

#define DRL_REWARD_ABS_ONE 0         /* agent/impala.py:45-46 */
#define DRL_REWARD_SOFT_ASYMMETRIC 1 /* agent/impala.py:47-49 */

/* Last error text of the calling thread ("" if none). */
const char* drl_last_error(void);
/* Library version string, e.g. "drl_b200 0.5 (sm_90a; ...)". */
const char* drl_version(void);
/* Number of CUDA devices visible (0 when there is none / no driver). */
int drl_device_count(void);

/* ------------------------------------------------------------------------------------------
 * Learner: replaces impala.Agent's learner graph + Agent.train (agent/impala.py:11-103,132-148)
 * over model/impala_actor_critic.py:33-118 and optimizer/vtrace.py:29-126.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_learner drl_learner;

typedef struct drl_learner_config {
  int32_t batch;              /* B trajectories per step on THIS device (config.json:130)      */
  int32_t trajectory;         /* T, 3..32 (config.json:136)                                      */
  int32_t height, width, channels; /* 84,84,4 -- only this geometry is supported (config.json:133) */
  int32_t num_action;         /* A, 2..32 (config.json:134)                                     */
  int32_t lstm_size;          /* 256 -- only this size is supported (config.json:137); see also `recurrent` */
  float discount_factor;      /* agent/impala.py:51                                             */
  float start_learning_rate;  /* agent/impala.py:96                                             */
  float end_learning_rate;
  double learning_frame;      /* decay_steps of tf.train.polynomial_decay                       */
  float baseline_loss_coef;   /* agent/impala.py:93                                             */
  float entropy_coef;
  float gradient_clip_norm;   /* agent/impala.py:98                                             */
  int32_t reward_clipping;    /* DRL_REWARD_*                                                   */
  int32_t device;             /* CUDA device ordinal                                            */
  int32_t num_slots;          /* device staging slots for stream-overlapped H2D (>=1, default 2) */
  int32_t use_cuda_graph;     /* 1: capture forward+backward(+apply) into CUDA graphs           */
  int32_t math_mode;          /* 0 = default (5); 1 = FP32 FFMA; 2 = wgmma 3xTF32; 3 = same, persistent kernels;
                                 5 = wgmma on bf16 hi/lo split operands (three products, fp32-grade) + bulk-fed
                                 LSTM weight gradient; any other value (4 included) is DRL_ERR_INVALID */
  int32_t recurrent;          /* 0 = the reference's learner: every step is one LSTM step from the (h, c) the actor
                                 recorded for it, no gradient through time.  1 = the LSTM runs through the T steps of
                                 each trajectory from the recorded state of step 0; after a done step the next step
                                 restarts from its recorded state; BPTT over the T - 2 steps with loss gradient, not
                                 across a done; the recorded states get no gradient (DESIGN.md section 21).  Same
                                 parameters, checkpoints and entry points; drl_learner_act stays one step.  Math
                                 modes 5 (default) and 2 only (1 and 3 -> DRL_ERR_INVALID).  The recurrent mode adds
                                 the named buffers "hin", "cin" (state each step read), "hout", "tc" (tanh c) for
                                 drl_learner_read_buffer.  Any other value -> DRL_ERR_INVALID, before any device
                                 lookup. */
} drl_learner_config;

/* Results of one step: the 4 floats Agent.train returns (agent/impala.py:144-148) + grad norm. */
typedef struct drl_step_out {
  float pi_loss;
  float baseline_loss;
  float entropy;
  float learning_rate;
  float grad_norm;   /* global norm before clipping (tf.clip_by_global_norm's second output) */
  float total_loss;  /* agent/impala.py:93 */
  int64_t step;      /* global_step AFTER this update (agent/impala.py:95,100) */
} drl_step_out;

/* impala.Agent.__init__ (agent/impala.py:11-103): allocates parameters (zeros), RMSProp slots
 * (ones, TF1 semantics), activations, staging slots, streams and events on cfg->device. */
int drl_learner_create(const drl_learner_config* cfg, drl_learner** out);
int drl_learner_destroy(drl_learner* h);

/* Number of learnable floats (4,153,267 for the reference geometry, SURVEY.md App. A.6). */
int drl_learner_param_count(const drl_learner* h, int64_t* n);
/* Flat float32 parameter vector in TF layouts / TF variable-creation order
 * (conv HWIO, dense [in,out], LSTM [in+h, 4*units] gate order i,j,f,o); replaces
 * global_variables_initializer / Saver.restore (agent/impala.py:105-109,114-116). */
int drl_learner_set_params(drl_learner* h, const float* host_flat, int64_t n);
int drl_learner_get_params(drl_learner* h, float* host_flat, int64_t n);      /* parameter_sync / Saver.save */
/* RMSProp "ms" slots (same flat layout) and global_step -- optimizer state of agent/impala.py:95-100. */
int drl_learner_set_opt_state(drl_learner* h, const float* host_ms_flat, int64_t n, int64_t step);
int drl_learner_get_opt_state(drl_learner* h, float* host_ms_flat, int64_t n, int64_t* step);
/* Gradient of total_loss (before clipping; summed over ranks if an all-reduce ran) -- parity tap
 * for optimizer.compute_gradients (agent/impala.py:98). */
int drl_learner_get_grads(drl_learner* h, float* host_flat, int64_t n);

/* Feed of Agent.train (agent/impala.py:134-142): asynchronous H2D of one batch-major batch
 * into device staging slot `slot` on the copy stream.  state u8 [B,T,H,W,C]; reward f32 [B,T];
 * action i32 [B,T]; done u8/bool [B,T]; behavior_policy f32 [B,T,A]; previous_action i32 [B,T];
 * initial_h, initial_c f32 [B,T,L].  The /255 normalisation (agent/impala.py:133) happens on
 * the device.  Host buffers must stay valid until the next drl_learner_wait / _step on the slot. */
int drl_learner_stage(drl_learner* h, int32_t slot,
                      const uint8_t* state, const float* reward, const int32_t* action,
                      const uint8_t* done, const float* behavior_policy,
                      const int32_t* previous_action, const float* initial_h, const float* initial_c);
/* The device trajectory queue (drl_traj_queue_create, below). */
typedef struct drl_traj_queue drl_traj_queue;
/* drl_learner_stage from a device trajectory queue: pops the oldest full batch (blocking like drl_ring_pop_batch;
 * a time-out is DRL_ERR_TIMEOUT and leaves the queue and the slot untouched), then on the copy stream waits for the
 * slot's last reader and the batch's commits, copies the batch device to device and hands the queue slot back to the
 * producers without a host wait.  The queue must have the learner's batch, trajectory, num_action, geometry and device
 * (DRL_ERR_INVALID otherwise). */
int drl_learner_stage_from_queue(drl_learner* h, int32_t slot, drl_traj_queue* queue, int32_t timeout_ms);

/* sess.run([pi_loss, baseline_loss, entropy, learning_rate, train_op]) (agent/impala.py:144-146):
 * forward, V-trace, losses, backward, global-norm clip, RMSProp, step += 1 on slot `slot`;
 * blocks until the scalars are on the host. */
int drl_learner_step(drl_learner* h, int32_t slot, drl_step_out* out);
/* Same, asynchronous: enqueue on the compute stream; drl_learner_wait collects the scalars. */
int drl_learner_step_async(drl_learner* h, int32_t slot);
int drl_learner_wait(drl_learner* h, drl_step_out* out);
/* (new) Result of the most recent drl_learner_step_async on `slot` (blocks until that step is done).  Every slot has
 * its own result record, so with two slots the host can keep two steps in flight and read step i-1 while step i runs. */
int drl_learner_wait_slot(drl_learner* h, int32_t slot, drl_step_out* out);

/* Data-parallel split of the step (SURVEY.md 8(e)): forward+backward leaves the local gradient
 * sum in the bucket; the caller all-reduces (SUM) `count` floats at `dev_ptr` across ranks on
 * `stream` (the bucket tail carries the 3 loss sums so one collective covers them); apply does
 * clip + RMSProp on the reduced bucket. */
int drl_learner_forward_backward(drl_learner* h, int32_t slot);
int drl_learner_grad_bucket(drl_learner* h, void** dev_ptr, int64_t* count);
int drl_learner_apply(drl_learner* h);          /* async; follow with drl_learner_wait */
/* (new) Device pointer of the bucket the update reads: the peer exchange's `reduced` buffer when that exchange is
 * on, else the gradient bucket itself (already all-reduced by the caller).  Same shape as drl_learner_grad_bucket.
 * Lets a harness compare the fused exchange with a library all-reduce of the saved local buckets (bench.py,
 * tests/test_gpu_multi.py). */
int drl_learner_reduced_bucket(drl_learner* h, void** dev_ptr, int64_t* count);
/* (new) Gradient exchange over NVLink peer memory, fused with the global-norm partials, INSTEAD of an all-reduce of
 * the bucket (one process per GPU on one node; buffers shared through CUDA IPC).  Every rank calls peer_export (128
 * bytes out: IPC handles of its bucket and of its exchange buffer), the ranks all-gather those blobs by any means
 * (torch.distributed in learner.py), then every rank calls peer_import with the world x 128 bytes in rank order.
 * From then on drl_learner_step / _step_async / _apply perform the exchange themselves inside the step's CUDA graph:
 * device-side barrier, each rank sums its slice of every rank's bucket in rank order and delivers it to every rank
 * (bit-identical replicas), barrier, clip + RMSProp.  Do not all-reduce the bucket as well.  All ranks must step in
 * lockstep; a rank that never arrives is reported by drl_learner_wait after a 20 s device-side time-out. */
int drl_learner_peer_export(drl_learner* h, void* handles, int64_t bytes);
int drl_learner_peer_import(drl_learner* h, int32_t rank, int32_t world, const void* all_handles, int64_t bytes);
/* Back to the local update (the caller all-reduces the bucket again); also the clean-up after a failed import. */
int drl_learner_peer_disable(drl_learner* h);
/* The handle's compute stream (cudaStream_t as void*), for ordering external work (NCCL). */
int drl_learner_stream(drl_learner* h, void** stream);

/* Forward only (no update): the learner-side values of build_network
 * (model/impala_actor_critic.py:71-118): policy [B,T,A] and value [B,T], batch-major, for all T
 * rows (first/middle/last are the slices [:, :-2], [:, 1:-1], [:, 2:]).  Host outputs. */
int drl_learner_forward(drl_learner* h, int32_t slot, float* policy, float* value);

/* Parity taps of the last step (agent/impala.py:68-80): vs, clipped_rho, vs_plus_1, pg_advantage,
 * each host float32 [B, T-2] batch-major.  NULL pointers are skipped. */
int drl_learner_taps(drl_learner* h, float* vs, float* clipped_rho, float* vs_plus_1, float* pg_advantage);

/* Debug/parity read of an internal activation by name into host memory (float32, device layout:
 * rows are TIME-MAJOR m = t*B + b).  Names: "a1" [M,20,20,32], "a2" [M,9,9,64], "a3" [M,3136],
 * "emb" [A,256], "h1","c1" [M,256], "logits","policy" [M,A], "value" [M].  n = element count. */
int drl_learner_read_buffer(drl_learner* h, const char* name, float* host_dst, int64_t n);

/* Actor-side shim of Agent.get_policy_and_action (agent/impala.py:118-130): n independent
 * single-step forwards.  state u8 [n,H,W,C]; previous_action i32 [n]; h,c f32 [n,L] ->
 * policy [n,A], h_out, c_out [n,L] (host).  n <= batch*trajectory. */
int drl_learner_act(drl_learner* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                    const float* h_in, const float* c_in, float* policy, float* h_out, float* c_out);

/* Measurement aid (bench.py roofline): runs ONE real step on a staged slot with a CUDA event recorded
 * on the compute stream before every kernel launch and returns per-launch device times.  names is a
 * '\n'-joined list (names_len bytes available), ms[i] the time from launch i to launch i+1. */
int drl_learner_profile_step(drl_learner* h, int32_t slot, char* names, int64_t names_len, float* ms,
                             int32_t max_kernels, int32_t* count);
/* Test aid: one plain GEMM C[M,N] = A*B on a chosen contraction core (1 = FP32 FFMA, 2 = wgmma 3xTF32, 5-8 = wgmma 16-bit split) and
 * operand-major combination, to validate shared-memory layouts / UMMA descriptors in isolation.
 * a_kmajor: A is [M,K] row-major (1) or [K,M] row-major (0); b_kmajor: B is [N,K] (1) or [K,N] (0).
 * C: `splits` slabs of [(M+1), N] floats (split-K partials; row M = column sums of B for N-major B). */
int drl_debug_gemm(int32_t core, int32_t bn, int32_t a_kmajor, int32_t b_kmajor, int32_t M, int32_t N,
                   int32_t K, int32_t splits, const float* A, const float* B, float* C);
/* Test aid: the IMPALA step's launch plan at B x T in math mode `mode` (needs the current device for its SM count):
 * out[0..2] = split-K count of the conv1 / conv2 / conv3 weight gradients, out[3] / out[4] = frames per CTA of the
 * persistent conv1 forward / weight-gradient kernels (math mode 5, else 0), out[5] = M tile of the 16-bit split core. */
int drl_debug_launch_plan(int32_t B, int32_t T, int32_t mode, int32_t* out);
/* Test aid: the launch plan of an Ape-X / A3C step over B transitions (forward rows 2B, backward rows B) in math mode 1
 * or 2: out[0] = split-K count of the first head layer (heads_l1_fwd), out[1..3] = split-K count of the conv1 / conv2 /
 * conv3 weight gradients. */
int drl_debug_apex_launch_plan(int32_t B, int32_t mode, int32_t* out);
/* Test aid: the launch plan of an R2D2 step over B sequences of S steps of C-channel frames (M = B*S rows) in math
 * mode 1 or 2 at lstm_size 64, 256 or 512 (others -> DRL_ERR_INVALID): out[0] = split-K count of the LSTM input
 * contraction (lstm_x_fwd, N = 4 lstm_size), out[1..3] = split-K count of the conv1 / conv2 / conv3 weight gradients
 * (conv1: the single-channel plan when C == 1), out[4] = sequences per cluster pass of the recurrence (0 at 64). */
int drl_debug_r2d2_launch_plan(int32_t B, int32_t S, int32_t C, int32_t mode, int32_t lstm_size, int32_t* out);
/* Test aid: CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor at the launch's block size and dynamic shared
 * memory) of the math-mode-5 kernels sized for two per SM: out[0] / out[1] = conv2 / conv3 forward, out[2] = conv2
 * data gradient. */
int drl_debug_gemm16_residency(int32_t* out);
/* Test aid: local memory per thread (bytes) of three math-mode-5 GEMMs of the IMPALA step: out[0] = LSTM forward,
 * out[1] = LSTM data gradient, out[2] = LSTM weight gradient.  A nonzero count means a wgmma accumulator left the
 * registers, which serialises the kernel's MMAs. */
int drl_debug_gemm16_local_bytes(int32_t* out);
/* Test aid: arm (dev_buf: device buffer of >= 8001 uint64, word 0 = entry count, zeroed by the caller) or disarm
 * (NULL) the kernel start-time trace: CTA 0 of every kernel of the step appends {globaltimer ns, grid size << 32 |
 * block size}.  Gives the true timeline of a CUDA-graph replay across both streams (tools/timeline.py). */
int drl_debug_trace(void* dev_buf);
/* Device-time of the last step's compute (CUDA events on the compute stream), milliseconds. */
int drl_learner_last_step_ms(drl_learner* h, float* ms);
/* Number of kernel launches one step issues (for bench.py's gpu_launches claim). */
int drl_learner_launches_per_step(const drl_learner* h, int32_t* n);

/* ------------------------------------------------------------------------------------------
 * IMPALA policy engine (new): the actor side of train_impala.py:132-194 (the actor loop's batched forward and
 * sampling; the loop itself is distributed_reinforcement_learning_b200/actor.py).  A forward-only handle that serves
 * Agent.get_policy_and_action (agent/impala.py:118-130) for up to 64 environments per call, on its own stream next to a
 * training learner, and takes the learner's parameters device to device (parameter_sync, agent/impala.py:111-112).
 * It holds no optimizer state, gradients or backward buffers.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_policy drl_policy;

typedef struct drl_policy_config {
  int32_t max_batch;                 /* 1..64 rows (environments) per drl_policy_act call             */
  int32_t height, width, channels;   /* 84,84,4 -- only this geometry is supported (as the learner)   */
  int32_t num_action;                /* A, 2..32                                                      */
  int32_t lstm_size;                 /* 256 -- only this size is supported                            */
  int32_t device;                    /* CUDA device ordinal                                           */
  int32_t use_cuda_graph;            /* 1: one CUDA graph per row count n (input copy + 5 kernels)    */
} drl_policy_config;

int drl_policy_create(const drl_policy_config* cfg, drl_policy** out);
int drl_policy_destroy(drl_policy* h);
/* Same inventory and flat TF order as drl_learner_param_count / _set_params / _get_params. */
int drl_policy_param_count(const drl_policy* h, int64_t* n);
int drl_policy_set_params(drl_policy* h, const float* host_flat, int64_t n);
int drl_policy_get_params(drl_policy* h, float* host_flat, int64_t n);
/* parameter_sync (agent/impala.py:111-112) without a host round trip: the snapshot is the learner's parameters after
 * all work enqueued on it so far (a step in flight included), copied device to device on the policy's stream; the
 * learner's next update waits for the copy.  The learner must be on the same device and have the same num_action
 * (DRL_ERR_INVALID otherwise); a learner in the failed state is DRL_ERR_STATE.  Returns without waiting for the copy. */
int drl_policy_sync_from_learner(drl_policy* h, drl_learner* learner);
/* Agent.get_policy_and_action (agent/impala.py:118-130) for n <= max_batch environments, with the sampling on the GPU.
 * state u8 [n,H,W,C]; previous_action i32 [n] in [0, A); h_in, c_in f32 [n,L]; uniform f64 [n] in [0, 1) or NULL ->
 * policy f32 [n,A] (the actor head's softmax), h_out, c_out f32 [n,L], action i32 [n].  Per row the action is the
 * number of entries of cdf = cumsum(float64(policy)) / cdf[A-1] that are <= uniform, clamped to A-1: exactly what
 * numpy's legacy RandomState.choice(A, p=policy) picks from u = random_sample().  Synchronous (the outputs are in the
 * caller's memory on return); any output pointer may be NULL; `action` without `uniform` is DRL_ERR_INVALID. */
int drl_policy_act(drl_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
                   const float* c_in, const double* uniform, int32_t* action, float* policy, float* h_out,
                   float* c_out);
/* Device time of the most recent drl_policy_act (input copy + kernels; CUDA events on the policy's stream), ms. */
int drl_policy_last_act_ms(drl_policy* h, float* ms);
/* Test aid: read of an internal buffer of the most recent act or recorder act (n rows) by name into host memory
 * (float32, device layout), after the engine's stream: "a1" [n,20,20,32], "a2" [n,9,9,64], "a3" [n,3136] (the conv
 * activations), "e1" [A,256] (relu of the first embedding layer), "table" [A,256] (the action-embedding table),
 * "zpart" [splits][n][N] (the per-split partial sums of the first skinny GEMM; drl_policy_buffer_dims gives splits and
 * N).  count = element count; a wrong count or an unknown name is DRL_ERR_INVALID, a read before the first act
 * DRL_ERR_STATE.  A policy server's serve is not an act here: it leaves n as it was and overwrites the buffers.  The
 * same holds for drl_r2d2_policy_read_buffer and drl_apex_policy_read_buffer. */
int drl_policy_read_buffer(drl_policy* h, const char* name, float* host_dst, int64_t count);
/* out[0] = n of the most recent act (0: none yet), out[1] = splits, out[2] = N of "zpart": IMPALA 16 and 1024, R2D2
 * 48 and 256, Ape-X 53 and 512 (value stream, then mean stream), A3C 53 and 256. */
int drl_policy_buffer_dims(drl_policy* h, int32_t* out);

/* Recorder: binds an engine to a device trajectory queue (drl_traj_queue_create below) for n <= max_batch rows, with
 * device staging of n trajectories of the queue's T steps (39 MB at n = 64, T = 20).  Queue and engine must be on the
 * same device, with the same num_action and the 84x84x4 / lstm 256 geometry, and n must fit the queue at once; all
 * DRL_ERR_INVALID otherwise.  Without a device, DRL_ERR_CUDA.  Destroy the recorder before its engine and queue. */
typedef struct drl_policy_recorder drl_policy_recorder;
int drl_policy_recorder_create(drl_policy* h, drl_traj_queue* queue, int32_t n, drl_policy_recorder** out);
int drl_policy_recorder_destroy(drl_policy_recorder* r);
/* drl_policy_act of the recorder's n rows (same inputs, outputs and results; `uniform` is required) that also records
 * step t of rows 0..n-1 on the device: the frame, previous action, h_in and c_in given, and the policy and action
 * computed.  Steps are recorded in order t = 0..T-1; an act after step T-1 is DRL_ERR_STATE until the commit.  With
 * use_cuda_graph one graph per recorder replays every step (the step reaches the kernels through the staged input).
 * drl_policy_recorder_reset discards the steps recorded since the last commit (an unroll abandoned half-way, e.g. when
 * an environment raised); the queue never saw them. */
int drl_policy_recorder_act(drl_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                            const float* h_in, const float* c_in, const double* uniform, int32_t* action,
                            float* policy, float* h_out, float* c_out);
int drl_policy_recorder_reset(drl_policy_recorder* r);
/* After step T-1 (DRL_ERR_STATE otherwise): reward f32 [n,T] and done u8 [n,T] complete the n trajectories, which are
 * appended to the queue in row order at n consecutive positions.  Blocks while those positions are not free
 * (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed otherwise).  Only reward and done are copied from the
 * host; the rest moves device to device on the engine's stream after the target slots' last readers, and the learner's
 * staging waits for it.  Returns without waiting for the copies; the next unroll starts at t = 0.  If enqueueing the
 * copies fails after the positions were reserved, the queue goes into a failed state instead of blocking forever: this
 * commit returns the CUDA error, and every later commit, stage or read of the queue returns DRL_ERR_STATE. */
int drl_policy_recorder_commit(drl_policy_recorder* r, const float* reward, const uint8_t* done, int32_t timeout_ms);

/* Policy server: one engine serving num_envs environments (1..256) that step in other processes, with each
 * environment's recurrent state and unfinished trajectory on the GPU.  The server binds one engine, one device
 * trajectory queue (drl_traj_queue_create below) and an exchange block the caller allocates in memory it shares with
 * the processes that step the environments.  It keeps a device state table (per environment: h and c f32 [256], the
 * previous action, and t, the step of the current unroll the next act records) and a device staging of one trajectory
 * per environment in the queue's field order.
 *
 * Exchange block (page-aligned, at least drl_policy_server_exchange_bytes(num_envs) bytes): num_envs report records,
 * then num_envs reply records, every field 16-byte aligned.  Before environment e is served, its report holds the
 * frame the next action is for, the uniform draw the action is sampled with (as drl_policy_act's `uniform`), the
 * reward and done flag the environment gave for its previous action, and `reset` = 1 when the episode restarted (the
 * previous action, h and c taken as 0) or it is the environment's first act.  After the serve its reply holds the
 * action and the largest probability of its policy. */
#define DRL_SERVER_REPORT_FRAME 0          /* u8 [84,84,4]  */
#define DRL_SERVER_REPORT_UNIFORM 28224    /* f64, in [0, 1) */
#define DRL_SERVER_REPORT_REWARD 28240     /* f32            */
#define DRL_SERVER_REPORT_DONE 28256       /* u8             */
#define DRL_SERVER_REPORT_RESET 28272      /* u8             */
#define DRL_SERVER_REPORT_BYTES 28288
#define DRL_SERVER_REPLY_ACTION 0          /* i32            */
#define DRL_SERVER_REPLY_MAX_PROB 16       /* f32            */
#define DRL_SERVER_REPLY_BYTES 32
typedef struct drl_policy_server drl_policy_server;
/* num_envs * (REPORT_BYTES + REPLY_BYTES) rounded up to 4096; DRL_ERR_INVALID for num_envs outside [1, 256] */
int drl_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes);
/* Registers the exchange block with CUDA (mapped, portable) until destroy.  Queue and engine must be on the same device
 * with the same num_action and the 84x84x4 / lstm 256 geometry, the queue must take min(num_envs, max_batch)
 * trajectories at once, and the block must be page-aligned and large enough; all DRL_ERR_INVALID otherwise.  Without
 * a device, DRL_ERR_CUDA.  Destroy the server before its engine and queue; after that the block may be registered
 * again. */
int drl_policy_server_create(drl_policy* h, drl_traj_queue* queue, int32_t num_envs, void* exchange,
                             int64_t exchange_bytes, drl_policy_server** out);
int drl_policy_server_destroy(drl_policy_server* s);
/* Serves the n <= max_batch distinct environments env_ids (any subset of [0, num_envs), any order; DRL_ERR_INVALID
 * otherwise) from their reports, in one act of the engine on its stream: the reward and done of each one's previous
 * step land in its staged trajectory, every trajectory whose step T-1 that completes is appended to the queue (in
 * env_ids order), then the act records step t of each environment and writes its reply.  No host thread copies frame
 * bytes: the kernels read the reports from the registered block.  Blocks while the queue has no room for the completed
 * trajectories (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed otherwise).  Synchronous: the replies
 * are written on return.  With use_cuda_graph one graph per n replays the kernels.  A failure after the queue
 * positions were reserved puts the queue into its failed state, as drl_policy_recorder_commit. */
int drl_policy_server_serve(drl_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms);

/* ------------------------------------------------------------------------------------------
 * R2D2 policy engine (new): the actor side of train_r2d2.py:167-251 (the actor loop itself is
 * distributed_reinforcement_learning_b200/actor.py: R2D2VectorActor).  A forward-only handle that serves
 * Agent.get_action (agent/r2d2.py:171-191) for up to 64 environments per call, on its own stream next to a training
 * R2D2 learner, and takes the learner's main-scope parameters device to device.  The explore decision and the random
 * action are drawn on the host (numpy's global stream, as the reference); the argmax and the selection run on the GPU.
 * It holds no target scope, optimizer state, gradients or backward buffers.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_r2d2_policy drl_r2d2_policy;

typedef struct drl_r2d2_policy_config {
  int32_t max_batch;                 /* 1..64 rows (environments) per drl_r2d2_policy_act call        */
  int32_t height, width, channels;   /* 84,84,1 or 84,84,4 (as drl_r2d2_create)                        */
  int32_t num_action;                /* A, 2..32                                                      */
  int32_t lstm_size;                 /* 64 -- only this size is supported (as the learner)            */
  int32_t device;                    /* CUDA device ordinal                                           */
  int32_t use_cuda_graph;            /* 1: one CUDA graph per row count n (input copy + kernels)      */
} drl_r2d2_policy_config;

int drl_r2d2_policy_create(const drl_r2d2_policy_config* cfg, drl_r2d2_policy** out);
int drl_r2d2_policy_destroy(drl_r2d2_policy* h);
/* The R2D2 learner's main-scope inventory and flat TF order (drl_r2d2_param_count / drl_r2d2_get_params(.., 0, ..)). */
int drl_r2d2_policy_param_count(const drl_r2d2_policy* h, int64_t* n);
int drl_r2d2_policy_set_params(drl_r2d2_policy* h, const float* host_flat, int64_t n);
int drl_r2d2_policy_get_params(drl_r2d2_policy* h, float* host_flat, int64_t n);
/* parameter_sync without a host round trip: the learner's main parameters after all work enqueued on it so far (a step
 * in flight included), copied device to device on the policy's stream; the learner's next update waits for the copy.
 * The learner must be on the same device and have the same num_action and channels, and lstm_size 64
 * (DRL_ERR_INVALID otherwise).
 * Returns without waiting for the copy. */
int drl_r2d2_policy_sync_from_learner(drl_r2d2_policy* h, struct drl_r2d2* learner);
/* Agent.get_action (agent/r2d2.py:171-191) for n <= max_batch environments.  state u8 [n,H,W,C]; previous_action i32
 * [n] in [0, A); h_in, c_in f32 [n,64]; explore_action i32 [n] or NULL -> q f32 [n,A] (value - mean of the main scope),
 * action i32 [n], q_action f32 [n] (= q[action]), h_out, c_out f32 [n,64].  Per row, explore_action -1 (or NULL) is the
 * greedy action, the first maximum of q (np.argmax); a value in [0, A) is taken as the action; anything else is
 * DRL_ERR_INVALID.  Synchronous (the outputs are in the caller's memory on return); any output pointer may be NULL. */
int drl_r2d2_policy_act(drl_r2d2_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const float* h_in, const float* c_in, const int32_t* explore_action, int32_t* action, float* q,
                        float* q_action, float* h_out, float* c_out);
/* Device time of the most recent drl_r2d2_policy_act (input copy + kernels; CUDA events on the policy's stream), ms. */
int drl_r2d2_policy_last_act_ms(drl_r2d2_policy* h, float* ms);
/* Test aids: as drl_policy_read_buffer and drl_policy_buffer_dims. */
int drl_r2d2_policy_read_buffer(drl_r2d2_policy* h, const char* name, float* host_dst, int64_t count);
int drl_r2d2_policy_buffer_dims(drl_r2d2_policy* h, int32_t* out);

/* ------------------------------------------------------------------------------------------
 * Device R2D2 sequence queue (new): R2D2FIFOQueue with its batch slots in GPU memory.  Producers are R2D2 policy
 * recorders (drl_r2d2_policy_recorder_commit), the consumer is drl_r2d2_replay_add_from_queue; a sequence never passes
 * through the host except its reward and done.  A record is one stored-state sequence in the replay memory's row layout:
 * state u8 [S,84,84,C], previous_action i32 [S], action i32 [S], h0 f32 [64], c0 f32 [64], reward f32 [S], done u8 [S]
 * (106,547 B at S = 15, C = 1).  Like the replay memory, it keeps only step 0 of the stored (h, c), the only step the
 * learner reads.  A slot holds `batch` sequences field-major, each field batch-major, so a slot is a learner minibatch
 * as it is.  capacity is rounded up as the ring's, plus one slot (9 slots, 15.3 MB at S = 15, C = 1, capacity 128,
 * batch 16).  Thread-safe: several recorders may commit while one learner thread ingests.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_r2d2_queue drl_r2d2_queue;
/* seq_len >= 2, channels 1 or 4, num_action in [2, 32] (DRL_ERR_INVALID otherwise, checked first), 1 <= batch <=
 * capacity; DRL_ERR_CUDA ("no CPU fallback") when `device` does not exist. */
int drl_r2d2_queue_create(int32_t seq_len, int32_t channels, int32_t num_action, int32_t capacity, int32_t batch,
                          int32_t device, drl_r2d2_queue** out);
int drl_r2d2_queue_destroy(drl_r2d2_queue* q);
/* sequences committed and not yet popped */
int drl_r2d2_queue_size(drl_r2d2_queue* q);
/* Synchronous copy of the k-th queued sequence (0 = the next to be popped) into host arrays; for tests.  previous_h
 * and previous_c are step 0 only, f32 [64] (an R2D2FIFOQueue record holds [S, 64]).  DRL_ERR_INVALID for k outside
 * [0, size), DRL_ERR_STATE while a commit into its slot is in progress. */
int drl_r2d2_queue_read(drl_r2d2_queue* q, int32_t k, uint8_t* state, int32_t* previous_action, int32_t* action,
                        float* previous_h, float* previous_c, float* reward, uint8_t* done);

/* R2D2 recorder: binds an R2D2 engine to a device R2D2 queue for n <= max_batch rows, with device staging of n
 * sequences (4.3 MB at n = 40, S = 15, C = 1).  Queue and engine must be on the same device with the same num_action
 * and channels, and n must fit the queue at once; all DRL_ERR_INVALID otherwise.  Without a device, DRL_ERR_CUDA.
 * Destroy the recorder before its engine and queue. */
typedef struct drl_r2d2_policy_recorder drl_r2d2_policy_recorder;
int drl_r2d2_policy_recorder_create(drl_r2d2_policy* h, drl_r2d2_queue* queue, int32_t n,
                                    drl_r2d2_policy_recorder** out);
int drl_r2d2_policy_recorder_destroy(drl_r2d2_policy_recorder* r);
/* drl_r2d2_policy_act of the recorder's n rows (same inputs, checks, outputs and results) that also records step t of
 * rows 0..n-1 on the device: the frame and previous action given, the action chosen, and at t = 0 h_in and c_in.
 * Steps are recorded in order t = 0..S-1; an act after step S-1 is DRL_ERR_STATE until the commit.  With use_cuda_graph
 * one graph per recorder replays every step.  drl_r2d2_policy_recorder_reset discards the steps recorded since the
 * last commit. */
int drl_r2d2_policy_recorder_act(drl_r2d2_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                                 const float* h_in, const float* c_in, const int32_t* explore_action, int32_t* action,
                                 float* q, float* q_action, float* h_out, float* c_out);
int drl_r2d2_policy_recorder_reset(drl_r2d2_policy_recorder* r);
/* After step S-1 (DRL_ERR_STATE otherwise): reward f32 [n,S] and done u8 [n,S] complete the n sequences, which are
 * appended to the queue in row order; otherwise as drl_policy_recorder_commit. */
int drl_r2d2_policy_recorder_commit(drl_r2d2_policy_recorder* r, const float* reward, const uint8_t* done,
                                    int32_t timeout_ms);

/* R2D2 policy server: one R2D2 engine serving num_envs environments (1..256) that step in other processes, with each
 * environment's recurrent state and unfinished sequence on the GPU (DESIGN.md section 17).  It binds one engine, one
 * device R2D2 queue and an exchange block as the IMPALA policy server does, and keeps a device state table (per
 * environment: h and c f32 [64], the previous action, and t, the step of the current sequence the next act records)
 * and a device staging of one sequence per environment in the queue's field order (106,547 B per environment at
 * S = 15, C = 1).
 *
 * Exchange block: the IMPALA server's record sizes and stride, so drl_policy_server_exchange_bytes sizes it; num_envs
 * report records, then num_envs reply records, every field 16-byte aligned.  Before environment e is served, its report
 * holds the frame the next action is for (84x84xC, the queue's C; the record keeps 84x84x4 bytes for it at either C),
 * the explore action (-1: the greedy action; a value in [0, A): that action, as drl_r2d2_policy_act's explore_action),
 * the reward and done flag the environment gave for its previous action, and `reset` = 1 when the episode restarted
 * (the previous action, h and c taken as 0) or it is the environment's first act.  After the serve its reply holds the
 * action and q_action (q of the main scope at the action). */
#define DRL_R2D2_SERVER_REPORT_FRAME 0          /* u8 [84,84,C]  */
#define DRL_R2D2_SERVER_REPORT_EXPLORE 28224    /* i32, in [-1, A) */
#define DRL_R2D2_SERVER_REPORT_REWARD 28240     /* f32            */
#define DRL_R2D2_SERVER_REPORT_DONE 28256       /* u8             */
#define DRL_R2D2_SERVER_REPORT_RESET 28272      /* u8             */
#define DRL_R2D2_SERVER_REPORT_BYTES 28288
#define DRL_R2D2_SERVER_REPLY_ACTION 0          /* i32            */
#define DRL_R2D2_SERVER_REPLY_Q_ACTION 16       /* f32            */
#define DRL_R2D2_SERVER_REPLY_BYTES 32
typedef struct drl_r2d2_policy_server drl_r2d2_policy_server;
/* Registers the exchange block with CUDA (mapped, portable) until destroy.  Queue and engine must be on the same device
 * with the same num_action and channels, the queue must take min(num_envs, max_batch) sequences at once, and the block
 * must be page-aligned and large enough; all DRL_ERR_INVALID otherwise.  Without a device, DRL_ERR_CUDA.  Destroy the
 * server before its engine and queue; after that the block may be registered again. */
int drl_r2d2_policy_server_create(drl_r2d2_policy* h, drl_r2d2_queue* queue, int32_t num_envs, void* exchange,
                                  int64_t exchange_bytes, drl_r2d2_policy_server** out);
int drl_r2d2_policy_server_destroy(drl_r2d2_policy_server* s);
/* Serves the n <= max_batch distinct environments env_ids (any subset of [0, num_envs), any order; DRL_ERR_INVALID
 * otherwise) from their reports, in one act of the engine on its stream: the reward and done of each one's previous
 * step land in its staged sequence, every sequence whose step S-1 that completes is appended to the queue (in env_ids
 * order), then the act records step t of each environment (frame, previous action, action; at t = 0 h and c) and
 * writes its reply.  The serve reads each explore action once from the block on the host; one outside [-1, A) is
 * DRL_ERR_INVALID naming the environment, returned before anything is reserved or launched: the state table, the
 * staging, the queue and every reply are as they were.  Blocks while the queue has no room for the completed sequences
 * (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed otherwise).  Synchronous: the replies are written on
 * return.  With use_cuda_graph one graph per n replays the kernels.  A failure after the queue positions were reserved
 * puts the queue into its failed state, as drl_policy_recorder_commit. */
int drl_r2d2_policy_server_serve(drl_r2d2_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms);

/* ------------------------------------------------------------------------------------------
 * Ape-X / A3C policy engine (new): the actor side of train_apex.py:157-231 and train_a3c.py:112-183 (the actor loops
 * themselves are distributed_reinforcement_learning_b200/actor.py: ApexVectorActor, A3CVectorActor).  A forward-only
 * handle that serves the family's get_policy_and_action (agent/apex.py:88-102, agent/a3c.py:109-119) for up to 64
 * environments per call, on its own stream next to a training learner, and takes the learner's parameters device to
 * device.  The two families share the network body and the learner handle (drl_a3c is drl_apex with algo 1), so one
 * engine serves both; only the action rule differs:
 *   algo 0 (Ape-X)  q = value - "mean"; the first maximum of q, or the row's explore action (epsilon drawn on the host)
 *   algo 1 (A3C)    policy = softmax(actor); numpy's RandomState.choice(A, p=policy) for the row's host uniform draw
 * It holds no target scope, optimizer state, gradients or backward buffers.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_apex_policy drl_apex_policy;
typedef struct drl_apex_policy drl_a3c_policy;

typedef struct drl_apex_policy_config {
  int32_t max_batch;                 /* 1..64 rows (environments) per act call                        */
  int32_t height, width, channels;   /* 84,84,4 only (as drl_apex_create / drl_a3c_create)            */
  int32_t num_action;                /* A, 2..32                                                      */
  int32_t algo;                      /* 0 = Ape-X (drl_apex_policy_act), 1 = A3C (drl_a3c_policy_act)  */
  int32_t device;                    /* CUDA device ordinal                                           */
  int32_t use_cuda_graph;            /* 1: one CUDA graph per row count n (input copy + kernels)      */
} drl_apex_policy_config;

int drl_apex_policy_create(const drl_apex_policy_config* cfg, drl_apex_policy** out);
int drl_apex_policy_destroy(drl_apex_policy* h);
/* The learner's one-network inventory and flat TF order (drl_apex_get_params(.., DRL_APEX_MAIN, ..) for Ape-X,
 * drl_a3c_get_params for A3C). */
int drl_apex_policy_param_count(const drl_apex_policy* h, int64_t* n);
int drl_apex_policy_set_params(drl_apex_policy* h, const float* host_flat, int64_t n);
int drl_apex_policy_get_params(drl_apex_policy* h, float* host_flat, int64_t n);
/* parameter_sync without a host round trip: the learner's main parameters after all work enqueued on it so far (a step
 * in flight included), copied device to device on the policy's stream; the learner's next update waits for the copy.
 * Takes a drl_apex* or a drl_a3c* (the same type).  The learner must be of the policy's algo, on the same device and
 * have the same num_action (DRL_ERR_INVALID otherwise).  Returns without waiting for the copy. */
int drl_apex_policy_sync_from_learner(drl_apex_policy* h, struct drl_apex* learner);
/* Ape-X get_policy_and_action (agent/apex.py:88-102) for n <= max_batch environments (algo 0 only).  state u8
 * [n,84,84,4]; previous_action i32 [n] in [0, A); explore_action i32 [n] or NULL -> q f32 [n,A] (value - mean),
 * action i32 [n], q_action f32 [n] (= q[action]).  Per row, explore_action -1 (or NULL) is the greedy action, the first
 * maximum of q (np.argmax); a value in [0, A) is taken as the action.  Synchronous; any output pointer may be NULL. */
int drl_apex_policy_act(drl_apex_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                        const int32_t* explore_action, int32_t* action, float* q, float* q_action);
/* A3C get_policy_and_action (agent/a3c.py:109-119) for n <= max_batch environments (algo 1 only).  state u8
 * [n,84,84,4]; previous_action i32 [n] in [0, A); uniform f64 [n] in [0, 1) -> policy f32 [n,A] (softmax of the actor
 * stream), action i32 [n] = min(searchsorted(cumsum(float64(policy)) / cdf[A-1], uniform, side='right'), A-1) -- what
 * numpy's RandomState.choice(A, p=policy) picks for that draw -- and prob_action f32 [n] (= policy[action]).
 * Synchronous; any output pointer may be NULL. */
int drl_a3c_policy_act(drl_a3c_policy* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                       const double* uniform, int32_t* action, float* policy, float* prob_action);
/* Device time of the most recent act call (input copy + kernels; CUDA events on the policy's stream), ms. */
int drl_apex_policy_last_act_ms(drl_apex_policy* h, float* ms);
/* Test aids: as drl_policy_read_buffer and drl_policy_buffer_dims (both algos). */
int drl_apex_policy_read_buffer(drl_apex_policy* h, const char* name, float* host_dst, int64_t count);
int drl_apex_policy_buffer_dims(drl_apex_policy* h, int32_t* out);

/* ------------------------------------------------------------------------------------------
 * Device A3C trajectory queue (new, DESIGN.md section 15): A3CFIFOQueue with its records in GPU memory.  Producers are
 * A3C policy recorders (drl_a3c_policy_recorder_commit, below), the consumer is drl_a3c_stage_from_queue; a record never
 * passes through the host.  A record is one actor unroll of T steps in the A3C learner's staging order (the Ape-X
 * queue's): frames u8 [2T,84,84,4] (the state rows, then the next_state rows), previous_action then action i32 [2T],
 * reward f32 [T], done u8 [T] (1,807,104 B at T = 32).  One record per slot.  An A3CFIFOQueue holds one record; this
 * queue takes a capacity (one recorder commit of n unrolls needs n free records at once), rounded as the other device
 * queues round theirs: it holds capacity + 1 records.  Thread-safe: several recorders may commit while one learner
 * thread stages.  A distinct type from drl_apex_queue, with the same record.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_a3c_queue drl_a3c_queue;
/* trajectory in [1, 512], num_action in [2, 32], capacity >= 1 (DRL_ERR_INVALID otherwise, checked first);
 * DRL_ERR_CUDA ("no CPU fallback") when `device` does not exist. */
int drl_a3c_queue_create(int32_t trajectory, int32_t num_action, int32_t capacity, int32_t device, drl_a3c_queue** out);
int drl_a3c_queue_destroy(drl_a3c_queue* q);
/* records committed and not yet staged */
int drl_a3c_queue_size(drl_a3c_queue* q);
/* Synchronous copy of the k-th queued record (0 = the next to be staged) into host arrays: state, next_state u8
 * [T,84,84,4], previous_action, action i32 [T], reward f32 [T], done u8 [T]; for tests.  DRL_ERR_INVALID for k outside
 * [0, size), DRL_ERR_STATE while a commit into its slot is in progress. */
int drl_a3c_queue_read(drl_a3c_queue* q, int32_t k, uint8_t* state, uint8_t* next_state, int32_t* previous_action,
                       int32_t* action, float* reward, uint8_t* done);

/* A3C recorder: binds an A3C engine (algo 1) to a device A3C queue for n <= max_batch rows, with device staging of n
 * unrolls (36.1 MB at n = 20, T = 32).  An Ape-X engine, another device, another num_action, or an n that cannot fit
 * the queue at once are DRL_ERR_INVALID.  Without a device, DRL_ERR_CUDA.  Destroy the recorder before its engine and
 * queue. */
typedef struct drl_a3c_policy_recorder drl_a3c_policy_recorder;
int drl_a3c_policy_recorder_create(drl_a3c_policy* h, drl_a3c_queue* queue, int32_t n, drl_a3c_policy_recorder** out);
int drl_a3c_policy_recorder_destroy(drl_a3c_policy_recorder* r);
/* drl_a3c_policy_act of the recorder's n rows (same inputs, checks, outputs and results) that also records step t of
 * rows 0..n-1 on the device: state row t (the frame given), previous_action[t], action[t] (the action sampled) and, for
 * t >= 1, next_state row t-1.  previous_next_state u8 [n,84,84,4] is what env.step returned at step t-1 (ignored, and
 * may be NULL, at t = 0).  A row whose previous_next_state equals its state (byte compare on the host) gets the device
 * copy of its frame; otherwise (an episode reset) its previous_next_state crosses PCIe.  Steps are recorded in order
 * t = 0..T-1; an act after step T-1 is DRL_ERR_STATE until the commit.  With use_cuda_graph one graph per recorder
 * replays every step.  drl_a3c_policy_recorder_reset discards the steps recorded since the last commit. */
int drl_a3c_policy_recorder_act(drl_a3c_policy_recorder* r, const uint8_t* state, const int32_t* previous_action,
                                const double* uniform, const uint8_t* previous_next_state, int32_t* action,
                                float* policy, float* prob_action);
int drl_a3c_policy_recorder_reset(drl_a3c_policy_recorder* r);
/* After step T-1 (DRL_ERR_STATE otherwise): reward f32 [n,T], done u8 [n,T] and next_state u8 [n,84,84,4] (the step
 * T-1 results) complete the n unrolls, which are appended to the queue in row order; the n frames are uploaded with
 * reward and done and land in next_state row T-1.  Otherwise as drl_policy_recorder_commit. */
int drl_a3c_policy_recorder_commit(drl_a3c_policy_recorder* r, const float* reward, const uint8_t* done,
                                   const uint8_t* next_state, int32_t timeout_ms);

/* A3C policy server: one A3C engine (algo 1) serving num_envs environments (1..256) that step in other processes, with
 * each environment's unfinished unroll on the GPU (DESIGN.md section 18).  It binds one engine, one device A3C queue and
 * an exchange block as the IMPALA policy server does, and keeps a device state table (per environment: the previous
 * action and t, the step of the current unroll the next act records) and a device staging of one unroll per
 * environment in the queue's record layout (1,806,752 B per environment at T = 32).
 *
 * Exchange block (page-aligned, at least drl_a3c_policy_server_exchange_bytes(num_envs) bytes): num_envs report
 * records, then num_envs reply records, every field 16-byte aligned.  Before environment e is served, its report holds
 * the frame the next action is for, the uniform draw the action is sampled with (as drl_a3c_policy_act's `uniform`),
 * the reward and done flag the environment gave for its previous action, and `reset` = 1 when the episode restarted
 * (the previous action taken as 0) or it is the environment's first act.  When `reset` follows a step, next_state holds
 * the frame env.step returned for the previous action (the frame to act on is then the new episode's first frame); the
 * server reads it only then.  After the serve its reply holds the action and max_prob = policy[action]. */
#define DRL_A3C_SERVER_REPORT_FRAME 0          /* u8 [84,84,4]  */
#define DRL_A3C_SERVER_REPORT_NEXT_STATE 28224 /* u8 [84,84,4]  */
#define DRL_A3C_SERVER_REPORT_UNIFORM 56448    /* f64, in [0, 1) */
#define DRL_A3C_SERVER_REPORT_REWARD 56464     /* f32            */
#define DRL_A3C_SERVER_REPORT_DONE 56480       /* u8             */
#define DRL_A3C_SERVER_REPORT_RESET 56496      /* u8             */
#define DRL_A3C_SERVER_REPORT_BYTES 56512
#define DRL_A3C_SERVER_REPLY_ACTION 0          /* i32            */
#define DRL_A3C_SERVER_REPLY_MAX_PROB 16       /* f32            */
#define DRL_A3C_SERVER_REPLY_BYTES 32
typedef struct drl_a3c_policy_server drl_a3c_policy_server;
/* num_envs * (REPORT_BYTES + REPLY_BYTES) rounded up to 4096; DRL_ERR_INVALID for num_envs outside [1, 256] */
int drl_a3c_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes);
/* Registers the exchange block with CUDA (mapped, portable) until destroy.  The engine must be an A3C engine (algo 1),
 * queue and engine on the same device with the same num_action, the queue must take min(num_envs, max_batch) records at
 * once, and the block must be page-aligned and large enough; all DRL_ERR_INVALID otherwise.  Without a device,
 * DRL_ERR_CUDA.  Destroy the server before its engine and queue; after that the block may be registered again. */
int drl_a3c_policy_server_create(drl_a3c_policy* h, drl_a3c_queue* queue, int32_t num_envs, void* exchange,
                                 int64_t exchange_bytes, drl_a3c_policy_server** out);
int drl_a3c_policy_server_destroy(drl_a3c_policy_server* s);
/* Serves the n <= max_batch distinct environments env_ids (any subset of [0, num_envs), any order; DRL_ERR_INVALID
 * otherwise) from their reports, in one act of the engine on its stream: the reward, done and next_state of each one's
 * previous step land in its staged unroll, every unroll whose step T-1 that completes is appended to the queue (in
 * env_ids order), then the act records step t of each environment (state, previous action, action) and writes its
 * reply.  The uniform is read on the device only; the action is clamped to [0, A) whatever its value.  Blocks while
 * the queue has no room for the completed unrolls (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed
 * otherwise).  Synchronous: the replies are written on return.  With use_cuda_graph one graph per n replays the
 * kernels.  A failure after the queue positions were reserved puts the queue into its failed state, as
 * drl_policy_recorder_commit. */
int drl_a3c_policy_server_serve(drl_a3c_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms);

/* ------------------------------------------------------------------------------------------
 * Stand-alone V-trace (optimizer/vtrace.py), host-pointer convenience forms + device forms.
 * ------------------------------------------------------------------------------------------ */
/* vtrace.from_importance_weights (optimizer/vtrace.py:71-103): time-major [T,B] float32 inputs,
 * bootstrap_value [B]; outputs vs, clipped_rhos [T,B].  clip_rho_threshold < 0 means None. */
int drl_vtrace_from_importance_weights(const float* log_rhos, const float* discounts,
                                       const float* rewards, const float* values,
                                       const float* bootstrap_value, int32_t T, int32_t B,
                                       float clip_rho_threshold, float* vs, float* clipped_rhos);
int drl_vtrace_from_importance_weights_dev(const float* log_rhos, const float* discounts,
                                           const float* rewards, const float* values,
                                           const float* bootstrap_value, int32_t T, int32_t B,
                                           float clip_rho_threshold, float* vs, float* clipped_rhos,
                                           void* stream);
/* vtrace.from_softmax (optimizer/vtrace.py:29-69): batch-major behavior/target softmax [B,T,A],
 * actions i32 [B,T], discounts/rewards/values/next_values f32 [B,T] -> vs, clipped_rho [B,T]. */
int drl_vtrace_from_softmax(const float* behavior_policy_softmax, const float* target_policy_softmax,
                            const int32_t* actions, const float* discounts, const float* rewards,
                            const float* values, const float* next_values, int32_t B, int32_t T,
                            int32_t A, float clip_rho_threshold, float* vs, float* clipped_rho);
int drl_vtrace_from_softmax_dev(const float* behavior_policy_softmax, const float* target_policy_softmax,
                                const int32_t* actions, const float* discounts, const float* rewards,
                                const float* values, const float* next_values, int32_t B, int32_t T,
                                int32_t A, float clip_rho_threshold, float* vs, float* clipped_rho,
                                void* stream);

/* The three loss sums of optimizer/vtrace.py:105-126 and log_probs_from_softmax_and_actions (:16-27)
 * in one pass over host arrays: softmax [B,T,A], actions i32 [B,T], advantages/vs/value f32 [B,T] ->
 * sums[3] = { -sum log(pi(a)+1e-8)*adv, 0.5*sum (vs-value)^2, sum pi*log(pi) }, log_probs [B,T]
 * (= log pi(a), no epsilon; may be NULL). */
int drl_vtrace_loss_sums(const float* softmax, const int32_t* actions, const float* advantages,
                         const float* vs, const float* value, int32_t B, int32_t T, int32_t A,
                         float* sums, float* log_probs);

/* ------------------------------------------------------------------------------------------
 * Trajectory ring: replaces buffer_queue.FIFOQueue (distributed_queue/buffer_queue.py:418-512).
 * A FIFO of `capacity` trajectories kept in pinned host memory, organised as batch slots of
 * `batch` trajectories in field-major order so that a popped batch is 8 contiguous [B, ...]
 * arrays ready for one async H2D each.  next_state is accepted by the Python shim and dropped
 * (the learner never reads it, train_impala.py:100-108).
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_ring drl_ring;

typedef struct drl_ring_batch {      /* views into the ring's pinned memory, valid until release */
  uint8_t* state;            /* [B,T,H,W,C] */
  float* reward;             /* [B,T]       */
  uint8_t* done;             /* [B,T]       */
  float* behavior_policy;    /* [B,T,A]     */
  int32_t* action;           /* [B,T]       */
  int32_t* previous_action;  /* [B,T]       */
  float* previous_h;         /* [B,T,L]     */
  float* previous_c;         /* [B,T,L]     */
  int32_t slot;              /* batch-slot index to pass to drl_ring_release */
} drl_ring_batch;

/* FIFOQueue.__init__ (buffer_queue.py:419-466).  capacity is rounded up to a multiple of batch
 * (+ one extra batch slot so producers can fill while the consumer holds one).  pinned=1 uses
 * cudaHostAlloc; if that fails (no device) it falls back to page-aligned malloc and *pinned=0. */
int drl_ring_create(int32_t trajectory, int32_t height, int32_t width, int32_t channels,
                    int32_t num_action, int32_t lstm_size, int32_t capacity, int32_t batch,
                    int32_t want_pinned, drl_ring** out);
int drl_ring_destroy(drl_ring* r);
int drl_ring_is_pinned(const drl_ring* r);
/* FIFOQueue.append_to_queue (buffer_queue.py:468-484): copies one trajectory in; blocks while the
 * ring is full (timeout_ms < 0: forever; DRL_ERR_TIMEOUT otherwise). */
int drl_ring_push(drl_ring* r, const uint8_t* state, const float* reward, const uint8_t* done,
                  const float* behavior_policy, const int32_t* action, const int32_t* previous_action,
                  const float* previous_h, const float* previous_c, int32_t timeout_ms);
/* FIFOQueue.sample_batch (buffer_queue.py:486-505): pops the oldest `batch` trajectories (FIFO
 * order) as one batch slot; blocks until a full batch is available. */
int drl_ring_pop_batch(drl_ring* r, drl_ring_batch* out, int32_t timeout_ms);
/* Hands a popped batch slot back to the producers. */
int drl_ring_release(drl_ring* r, int32_t slot);
/* FIFOQueue.get_size (buffer_queue.py:507-509): trajectories enqueued and not yet popped. */
int drl_ring_size(drl_ring* r);

/* ------------------------------------------------------------------------------------------
 * Device trajectory queue (new): the ring's FIFO with its batch slots in GPU memory.  Producers are policy recorders
 * (drl_policy_recorder_commit), the consumer is drl_learner_stage_from_queue; a batch never passes through the host.
 * A slot holds `batch` trajectories field-major in the learner's batch-major staging layout, so staging a batch is
 * eight device-to-device copies.  capacity is rounded up as the ring's, plus one slot (97 MB at T = 20, A = 18,
 * capacity 128, batch 32).  Thread-safe: several recorders may commit while one learner stages.
 * ------------------------------------------------------------------------------------------ */
/* (drl_traj_queue is declared with the learner above.)  DRL_ERR_CUDA ("no CPU fallback") when `device` does not exist. */
int drl_traj_queue_create(int32_t trajectory, int32_t height, int32_t width, int32_t channels, int32_t num_action,
                          int32_t lstm_size, int32_t capacity, int32_t batch, int32_t device, drl_traj_queue** out);
int drl_traj_queue_destroy(drl_traj_queue* q);
/* trajectories committed and not yet popped by a learner (as drl_ring_size) */
int drl_traj_queue_size(drl_traj_queue* q);
/* Synchronous copy of the k-th queued trajectory (0 = the next to be popped) into host arrays laid out as
 * drl_ring_push takes them; for tests.  DRL_ERR_INVALID for k outside [0, size), DRL_ERR_STATE while a commit into
 * its slot is in progress. */
int drl_traj_queue_read(drl_traj_queue* q, int32_t k, uint8_t* state, float* reward, uint8_t* done,
                        float* behavior_policy, int32_t* action, int32_t* previous_action, float* previous_h,
                        float* previous_c);

/* ------------------------------------------------------------------------------------------
 * Ape-X DQN learner (SURVEY.md section 8(f) row 2, BASELINE.json config 4): replaces apex.Agent's learner graph
 * (agent/apex.py:12-76) over model/apex_value.py:4-66 (dueling network: q = value stream - "mean" stream, evaluated
 * as main(s, prev_a), main(s', a), target(s', a)), optimizer/dqn.py:3-7 and TF1 Adam.  The three network
 * evaluations run as ONE main-network forward over 2B rows [s ; s'] plus one target-network forward over B rows;
 * only the first B rows are differentiated.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_apex drl_apex;

#define DRL_APEX_MAIN 0
#define DRL_APEX_TARGET 1

typedef struct drl_apex_config {
  int32_t batch;              /* B transitions per step (config.json:154)                               */
  int32_t height, width, channels; /* 84,84,4 -- only this geometry is supported (config.json:156)      */
  int32_t num_action;         /* A, 2..32 (config.json:157)                                             */
  float discount_factor;      /* agent/apex.py:43                                                       */
  float start_learning_rate;  /* agent/apex.py:71                                                       */
  float end_learning_rate;
  double learning_frame;      /* decay_steps of tf.train.polynomial_decay                               */
  float gradient_clip_norm;   /* agent/apex.py:74                                                       */
  int32_t reward_clipping;    /* DRL_REWARD_ABS_ONE clips to [-1,1]; anything else passes the reward through
                                 (agent/apex.py:38-41)                                                  */
  int32_t device;             /* CUDA device ordinal                                                    */
  int32_t num_slots;          /* device staging slots for stream-overlapped H2D (>=1, default 2)        */
  int32_t use_cuda_graph;     /* 1: capture the whole step into one CUDA graph per slot                 */
  int32_t math_mode;          /* 0 = default (2); 1 = FP32 FFMA; 2 = wgmma 3xTF32 convolutions          */
} drl_apex_config;

typedef struct drl_apex_out {
  float loss;           /* value_loss = mean(is_weight * (target_value - state_action_value)^2), agent/apex.py:63-65 */
  float learning_rate;  /* agent/apex.py:71 */
  float grad_norm;      /* global norm before clipping (agent/apex.py:74) */
  int64_t step;         /* global_step AFTER this update (agent/apex.py:70,75) */
} drl_apex_out;

/* apex.Agent.__init__ (agent/apex.py:12-76): parameters of 'main' and 'target' (zeros until set), Adam slots m, v
 * (zeros), beta powers (0.9, 0.999), activations, staging slots, streams on cfg->device. */
int drl_apex_create(const drl_apex_config* cfg, drl_apex** out);
int drl_apex_destroy(drl_apex* h);
/* Learnable floats of ONE network (main and target have the same inventory). */
int drl_apex_param_count(const drl_apex* h, int64_t* n);
/* Flat float32 vector in TF layouts / TF variable-creation order of the scope ({model}/main or {model}/target):
 * conv2d x3 (HWIO), dense x2 (action embedding), dense x3 (value stream), dense x3 ("mean" stream); which =
 * DRL_APEX_MAIN / DRL_APEX_TARGET.  Replaces global_variables_initializer / Saver (agent/apex.py:76,84-86). */
int drl_apex_set_params(drl_apex* h, int32_t which, const float* host_flat, int64_t n);
int drl_apex_get_params(drl_apex* h, int32_t which, float* host_flat, int64_t n);
/* Adam slots of the main network, global_step, beta1_power, beta2_power (agent/apex.py:72). */
int drl_apex_set_opt_state(drl_apex* h, const float* host_m, const float* host_v, int64_t n, int64_t step,
                           float beta1_power, float beta2_power);
int drl_apex_get_opt_state(drl_apex* h, float* host_m, float* host_v, int64_t n, int64_t* step,
                           float* beta1_power, float* beta2_power);
/* Gradient of value_loss w.r.t. the main network, before clipping (parity tap of compute_gradients, agent/apex.py:73). */
int drl_apex_get_grads(drl_apex* h, float* host_flat, int64_t n);
/* Agent.target_to_main (agent/apex.py:78-79 -> utils.main_to_target, utils.py:27-32): despite its name it assigns
 * target <- main. */
int drl_apex_target_to_main(drl_apex* h);

/* Feed of Agent.distributed_train (agent/apex.py:135-149): asynchronous H2D into staging slot `slot`.
 * state, next_state u8 [B,H,W,C] (the /255 of :136-137 happens on the device); previous_action, action i32 [B];
 * reward f32 [B]; done u8/bool [B]; is_weight f32 [B] or NULL (= ones: Agent.train, agent/apex.py:156-168). */
int drl_apex_stage(drl_apex* h, int32_t slot, const uint8_t* state, const uint8_t* next_state,
                   const int32_t* previous_action, const int32_t* action, const float* reward,
                   const uint8_t* done, const float* is_weight);
/* sess.run([value_loss, target_value, state_action_value, train_op]) (agent/apex.py:139-149): forward x3, TD target,
 * weighted squared loss, backward through main(s), global-norm clip, Adam, step += 1.  td_error (host, [B], may be
 * NULL) receives |target_value - state_action_value| from BEFORE the update (agent/apex.py:151): the new priorities. */
int drl_apex_step(drl_apex* h, int32_t slot, drl_apex_out* out, float* td_error);
int drl_apex_step_async(drl_apex* h, int32_t slot);
int drl_apex_wait(drl_apex* h, drl_apex_out* out, float* td_error);
/* (new) Data-parallel step in two halves (one process per GPU, each rank feeds its own B transitions): forward + TD +
 * backward into the gradient bucket [padded grads | loss scalars] -> the CALLER all-reduces (SUM) the bucket on the
 * learner's stream (drl_apex_stream) -> clip + Adam on bucket * grad_scale.  value_loss is a batch MEAN
 * (agent/apex.py:65), so grad_scale = 1 / world_size makes the update that of the undivided global batch. */
int drl_apex_forward_backward(drl_apex* h, int32_t slot);
int drl_apex_grad_bucket(drl_apex* h, void** dev_ptr, int64_t* count);
int drl_apex_apply(drl_apex* h, float grad_scale);   /* async; follow with drl_apex_wait */
/* Agent.get_td_error (agent/apex.py:116-133): forward only, n <= batch transitions -> |target - q(s,a)| [n]. */
int drl_apex_td_error(drl_apex* h, int32_t n, const uint8_t* state, const uint8_t* next_state,
                      const int32_t* previous_action, const int32_t* action, const float* reward,
                      const uint8_t* done, float* td_error);
/* Agent.get_policy_and_action without the epsilon-greedy draw (agent/apex.py:88-102): main_q_value [n, A] for
 * n <= 2*batch (state, previous_action) pairs. */
int drl_apex_act(drl_apex* h, int32_t n, const uint8_t* state, const int32_t* previous_action, float* q_value);
/* Parity taps of the most recent step / td_error call over its n rows (agent/apex.py:45-61): main_q_value,
 * next_main_q_value, target_q_value [n, A]; target_value, state_action_value [n].  Any pointer may be NULL. */
int drl_apex_taps(drl_apex* h, float* main_q, float* next_main_q, float* target_q, float* target_value,
                  float* state_action_value);
/* Debug/parity: copy a named device buffer of the MAIN network's last forward to the host.  Names: a1 a2 a3 e1 emb
 * hid1 hid2 (rows = 2n: [s ; s']), da1 da2 da3 (rows = n). */
int drl_apex_read_buffer(drl_apex* h, const char* name, float* host_dst, int64_t n);
/* Per-launch device times of one real step (CUDA events around every launch, serial). */
int drl_apex_profile_step(drl_apex* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels,
                          int32_t* count);
int drl_apex_last_step_ms(drl_apex* h, float* ms);
/* The learner's compute stream (cudaStream_t), for callers that time or order work against it. */
int drl_apex_stream(drl_apex* h, void** stream);
int drl_apex_launches_per_step(const drl_apex* h, int32_t* n);

/* ------------------------------------------------------------------------------------------
 * Prioritized replay index (host): replaces buffer_queue.SumTree / Memory (distributed_queue/buffer_queue.py:326-416)
 * -- float64 sum tree with the reference's arithmetic order (bit-identical totals), priorities (|td| + 0.001)^0.6,
 * stratified sampling, importance weights (n_entries * p / total)^-beta / max, beta 0.4 -> 1 by +0.001 per sample
 * call.  The transitions themselves stay with the caller (the Python shim keeps them, as the reference does); the
 * uniform draws of random.uniform(a, b) are passed in as u01 in [0,1) so that sampling is reproducible.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_per drl_per;
int drl_per_create(int64_t capacity, drl_per** out);
int drl_per_destroy(drl_per* p);
/* Memory.add (buffer_queue.py:386-388): stores priority (error + e)^a at the write cursor; returns the data index
 * the caller must store the transition at (SumTree.add, :351-359). */
int drl_per_add(drl_per* p, double error, int64_t* data_index);
/* Memory.sample (buffer_queue.py:390-411): n strata; tree_index[i] (SumTree.get's idx), data_index[i],
 * priority[i], is_weight[i]; also advances beta. */
int drl_per_sample(drl_per* p, int32_t n, const double* u01, int64_t* tree_index, int64_t* data_index,
                   double* priority, double* is_weight);
/* Memory.update (buffer_queue.py:413-415): tree_index as returned by drl_per_sample. */
int drl_per_update(drl_per* p, int64_t tree_index, double error);
int drl_per_total(const drl_per* p, double* total);      /* SumTree.total (:348-349) */
int drl_per_size(const drl_per* p, int64_t* n_entries);  /* SumTree.n_entries */
int drl_per_beta(const drl_per* p, double* beta);

/* ------------------------------------------------------------------------------------------
 * Ape-X prioritized replay memory on the device (DESIGN.md section 10): buffer_queue.Memory with the transitions in HBM
 * (state, next_state u8 [capacity,84,84,4]; previous_action, action i32; reward f32; done u8; zero-initialised), the
 * float64 sum tree on the device, and the learner loop of train_apex.py:82-155 -- ingest, sample, minibatch gather,
 * step, priority update -- as kernels on the learner's compute stream.  Same constants and arithmetic as drl_per_*
 * (e = 0.001, a = 0.6, beta 0.4 -> 1 by +0.001 per sample); the uniforms of random.uniform(a, b) come from the caller.
 * The memory outlives any learner: every call that uses one takes a drl_apex* (Ape-X, not A3C, on the memory's
 * device) and orders itself after the memory's previous work on whichever stream that ran.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_apex_replay drl_apex_replay;
/* capacity in [2, 2^31]: 56 KB of device memory per transition (5.6 GB at the reference's 1e5). */
int drl_apex_replay_create(int32_t device, int64_t capacity, drl_apex_replay** out);
int drl_apex_replay_destroy(drl_apex_replay* r);
/* Memory.add for n transitions in order at the write cursor (wrapping).  error == NULL: the priorities are the
 * learner's |td| of these transitions (agent/apex.py:116-133), computed on the device and never copied to the host;
 * then 1 <= n <= the learner's batch.  Otherwise error [n] are the caller's and learner may be NULL.  Does not wait
 * for the learner's compute stream. */
int drl_apex_replay_add(drl_apex_replay* r, drl_apex* learner, int32_t n, const uint8_t* state,
                        const uint8_t* next_state, const int32_t* previous_action, const int32_t* action,
                        const float* reward, const uint8_t* done, const double* error);
/* Memory.sample(B) with the caller's uniforms u01 [B] (B = the learner's batch) -> gather into staging slot `slot` ->
 * the learner's step on that slot -> Memory.update of the sampled leaves with the step's |td|.  Asynchronous:
 * drl_apex_wait returns the loss and the priorities once the update has run.  DRL_ERR_STATE on an empty memory. */
int drl_apex_replay_step_async(drl_apex_replay* r, drl_apex* learner, int32_t slot, const double* u01);
/* The device kernels without a learner (tests, callers with their own loop); synchronous.  sample is Memory.sample
 * (drl_per_sample's outputs, advances beta); update is Memory.update of n leaves in order. */
int drl_apex_replay_sample(drl_apex_replay* r, int32_t n, const double* u01, int64_t* tree_index,
                           int64_t* data_index, double* priority, double* is_weight);
int drl_apex_replay_update(drl_apex_replay* r, int32_t n, const int64_t* tree_index, const double* error);
/* The draws of the most recent sample (or step): tree_index, priority, is_weight [n]; any pointer may be NULL. */
int drl_apex_replay_last_sample(drl_apex_replay* r, int64_t* tree_index, double* priority, double* is_weight);
/* Rows [data_index, data_index + n) of the storage; any pointer may be NULL. */
int drl_apex_replay_read(drl_apex_replay* r, int64_t data_index, int32_t n, uint8_t* state, uint8_t* next_state,
                         int32_t* previous_action, int32_t* action, float* reward, uint8_t* done);
int drl_apex_replay_total(drl_apex_replay* r, double* total);      /* SumTree.total */
int drl_apex_replay_size(drl_apex_replay* r, int64_t* n_entries);  /* SumTree.n_entries */
int drl_apex_replay_beta(drl_apex_replay* r, double* beta);

/* ------------------------------------------------------------------------------------------
 * Device Ape-X transition queue (new, DESIGN.md section 14): ApexFIFOQueue with its records in GPU memory.  Producers
 * are Ape-X actor buffers (drl_apex_actor_buffer_push, below), the consumer is drl_apex_replay_add_from_queue; a record
 * never passes through the host.  A record is one local-buffer sample of T transitions, and a slot holds one record in
 * the learner's ApexIn order: frames u8 [2T,84,84,4] (the state rows, then the next_state rows), previous_action then
 * action i32 [2T], reward f32 [T], done u8 [T] (1,807,104 B at T = 32).  capacity is rounded as the other device
 * queues round it: capacity + 1 slots (59.6 MB at T = 32, capacity 32), so the queue holds one record more than an
 * ApexFIFOQueue of the same queue_size.  Thread-safe: several buffers may push while one learner thread ingests.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_apex_queue drl_apex_queue;
/* trajectory in [1, 512], num_action in [2, 32], capacity >= 1 (DRL_ERR_INVALID otherwise, checked first);
 * DRL_ERR_CUDA ("no CPU fallback") when `device` does not exist. */
int drl_apex_queue_create(int32_t trajectory, int32_t num_action, int32_t capacity, int32_t device,
                          drl_apex_queue** out);
int drl_apex_queue_destroy(drl_apex_queue* q);
/* records pushed and not yet popped */
int drl_apex_queue_size(drl_apex_queue* q);
/* Synchronous copy of the k-th queued record (0 = the next to be popped) into host arrays: state, next_state u8
 * [T,84,84,4], previous_action, action i32 [T], reward f32 [T], done u8 [T]; for tests.  DRL_ERR_INVALID for k outside
 * [0, size), DRL_ERR_STATE while a push into its slot is in progress. */
int drl_apex_queue_read(drl_apex_queue* q, int32_t k, uint8_t* state, uint8_t* next_state, int32_t* previous_action,
                        int32_t* action, float* reward, uint8_t* done);

/* Ape-X actor buffers (new, DESIGN.md section 14): the n LocalBuffer(capacity)s of one vector actor in GPU memory,
 * n * capacity rows in the replay memory's field layout, 56,461 B per row (11.3 GB at 20 environments x 1e4, 36 GB at
 * 64).  All n environments append in lockstep, so one length describes every buffer; deque index j of environment e is
 * the transition collections.deque(maxlen=capacity) would hold at index j.  Work runs on the buffer's own stream.
 * Thread-safe, but one actor thread is expected to own a buffer. */
typedef struct drl_apex_actor_buffer drl_apex_actor_buffer;
/* n >= 1, capacity >= 2, num_action in [2, 32] (DRL_ERR_INVALID, checked first); DRL_ERR_CUDA without the device. */
int drl_apex_actor_buffer_create(int32_t n, int32_t capacity, int32_t num_action, int32_t device,
                                 drl_apex_actor_buffer** out);
int drl_apex_actor_buffer_destroy(drl_apex_actor_buffer* b);
/* LocalBuffer.append for all n environments at once (n must be the buffer's): state, next_state u8 [n,84,84,4];
 * previous_action, action i32 [n] in [0, num_action) (DRL_ERR_INVALID otherwise, nothing changed); reward f32 [n]; done
 * u8 [n].  All of next_state crosses PCIe; a row's state only when it differs from the same environment's previous
 * next_state (otherwise the device copies that row).  One H2D from a pinned block, then one kernel. */
int drl_apex_actor_buffer_append(drl_apex_actor_buffer* b, int32_t n, const uint8_t* state, const uint8_t* next_state,
                                 const int32_t* previous_action, const int32_t* action, const float* reward,
                                 const uint8_t* done);
/* LocalBuffer.sample(T) of environment `env` with the draws given, then ApexFIFOQueue.append_to_queue: order i32 [T]
 * (T = the queue's) are deque indices in [0, size), checked on the host.  Reserves one queue position without holding
 * the buffer's lock, blocking while the queue is full (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed
 * otherwise), then gathers the rows into the slot on the device.  The queue's num_action and device must be the
 * buffer's (DRL_ERR_INVALID).  A failure after the reservation puts the queue into its failed state. */
int drl_apex_actor_buffer_push(drl_apex_actor_buffer* b, drl_apex_queue* queue, int32_t env, const int32_t* order,
                               int32_t timeout_ms);
/* the deque length (the same for every environment) */
int drl_apex_actor_buffer_size(drl_apex_actor_buffer* b, int64_t* len);
/* Synchronous copy of deque index j of environment env (one transition, the append's fields); for tests. */
int drl_apex_actor_buffer_read(drl_apex_actor_buffer* b, int32_t env, int64_t j, uint8_t* state, uint8_t* next_state,
                               int32_t* previous_action, int32_t* action, float* reward, uint8_t* done);
/* Ape-X policy server: one Ape-X engine (algo 0) serving num_envs environments (1..256) that step in other processes,
 * with each environment's LocalBuffer on the GPU (DESIGN.md section 19).  It binds one engine, one device Ape-X queue
 * and an exchange block as the other policy servers do, and keeps a device table (per environment: the previous action
 * and the ring row of the transition still waiting for its reward) and one ring of capacity + 1 rows per environment in
 * the replay memory's row layout (56,461 B per row: 565 MB per environment at capacity 1e4).  Deque index j of
 * environment e is ring row (appended - len + j) mod (capacity + 1), with appended and len kept on the host; the spare
 * row holds the pending transition, so it never overwrites a row the deque holds.
 *
 * Exchange block (page-aligned, at least drl_apex_policy_server_exchange_bytes(num_envs) bytes): num_envs report
 * records, then num_envs reply records, every field 16-byte aligned.  Before environment e is served, its report holds
 * the frame the next action is for, the explore action (as drl_apex_policy_act's explore_action: -1 greedy, otherwise
 * the action), the reward and done flag the environment gave for its previous action, `reset` = 1 when the episode
 * restarted (the previous action taken as 0) or it is the environment's first act, and, when the buffer's length after
 * this serve's append exceeds 3 T, the sample order: T deque indices in [0, length) (LocalBuffer.sample's
 * np.random.permutation(length)[:T]).  When `reset` follows a step, next_state holds the frame env.step returned for the
 * previous action; the server reads it only then.  After the serve its reply holds the action and q_action = q[action]. */
#define DRL_APEX_SERVER_REPORT_FRAME 0          /* u8 [84,84,4]        */
#define DRL_APEX_SERVER_REPORT_NEXT_STATE 28224 /* u8 [84,84,4]        */
#define DRL_APEX_SERVER_REPORT_EXPLORE 56448    /* i32, in [-1, A)     */
#define DRL_APEX_SERVER_REPORT_REWARD 56464     /* f32                 */
#define DRL_APEX_SERVER_REPORT_DONE 56480       /* u8                  */
#define DRL_APEX_SERVER_REPORT_RESET 56496      /* u8                  */
#define DRL_APEX_SERVER_REPORT_ORDER 56512      /* i32 [512], first T  */
#define DRL_APEX_SERVER_REPORT_BYTES 58560
#define DRL_APEX_SERVER_REPLY_ACTION 0          /* i32                 */
#define DRL_APEX_SERVER_REPLY_Q_ACTION 16       /* f32                 */
#define DRL_APEX_SERVER_REPLY_BYTES 32
typedef struct drl_apex_policy_server drl_apex_policy_server;
/* num_envs * (REPORT_BYTES + REPLY_BYTES) rounded up to 4096; DRL_ERR_INVALID for num_envs outside [1, 256] */
int drl_apex_policy_server_exchange_bytes(int32_t num_envs, int64_t* bytes);
/* Registers the exchange block with CUDA (mapped, portable) until destroy.  The engine must be an Ape-X engine (algo 0),
 * queue and engine on the same device with the same num_action, capacity > 3 T (T = the queue's trajectory), the queue
 * must take min(num_envs, max_batch) records at once, and the block must be page-aligned and large enough; all
 * DRL_ERR_INVALID otherwise.  Without a device, or when the rings do not fit, DRL_ERR_CUDA with nothing left allocated.
 * Destroy the server before its engine and queue; after that the block may be registered again. */
int drl_apex_policy_server_create(drl_apex_policy* h, drl_apex_queue* queue, int32_t num_envs, int32_t capacity,
                                  void* exchange, int64_t exchange_bytes, drl_apex_policy_server** out);
int drl_apex_policy_server_destroy(drl_apex_policy_server* s);
/* Serves the n <= max_batch distinct environments env_ids (any subset of [0, num_envs), any order; DRL_ERR_INVALID
 * otherwise) from their reports, in one act of the engine on its stream: each one's pending transition is completed
 * with the reward, done and next_state of its previous step (LocalBuffer.append), every environment whose length is
 * then > 3 T pushes its sample of T transitions to the queue (in env_ids order), then the act writes the new pending
 * transition (state, previous action, action) and the reply.  The host reads each explore action and each pushing
 * environment's T order entries once and checks them ([-1, A), [0, length)); a bad value is DRL_ERR_INVALID naming the
 * environment, with nothing reserved, launched or changed.  Blocks while the queue has no room for the pushed records
 * (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed otherwise).  Synchronous: the replies are written on
 * return.  With use_cuda_graph one graph per (n, whether any environment pushes) replays the kernels.  A failure after
 * the queue positions were reserved puts the queue into its failed state, as drl_policy_recorder_commit. */
int drl_apex_policy_server_serve(drl_apex_policy_server* s, int32_t n, const int32_t* env_ids, int32_t timeout_ms);
/* Synchronous copy of deque index j of environment env's ring (one transition: the fields
 * drl_apex_actor_buffer_read returns); DRL_ERR_INVALID outside [0, num_envs) x [0, length).  For tests. */
int drl_apex_policy_server_read(drl_apex_policy_server* s, int32_t env, int64_t j, uint8_t* state, uint8_t* next_state,
                                int32_t* previous_action, int32_t* action, float* reward, uint8_t* done);
/* drl_apex_replay_add of the oldest record of a device Ape-X queue (train_apex.py:94-116 without a host copy): pops it
 * without holding the memory's or the learner's lock, blocking while the queue is empty (timeout_ms < 0: forever;
 * DRL_ERR_TIMEOUT with nothing changed otherwise), then, on the learner's compute stream, the learner's |td| of the T
 * transitions read from the queue slot, the store and the priority update; the slot goes back to the producers after
 * them, also when enqueueing fails.  The learner must be an Ape-X (not A3C) handle on the memory's device with the
 * queue's num_action and device, and T at most its batch (DRL_ERR_INVALID).  Does not wait for the compute stream. */
int drl_apex_replay_add_from_queue(drl_apex_replay* r, drl_apex* learner, drl_apex_queue* queue, int32_t timeout_ms);

/* ------------------------------------------------------------------------------------------
 * R2D2 learner (SURVEY.md section 8(f) row 3, BASELINE.json config 5): replaces r2d2.Agent's learner graph
 * (agent/r2d2.py:13-95) over model/r2d2_lstm.py:28-116 (conv stack + action embedding + ONE LSTMCell, unrolled seq_len
 * steps per scope from a stored (h, c) with the carried state multiplied by (1 - done) after every step; dense 128;
 * q = value - "mean"), optimizer/burn_in.py:23-32 (value-function rescaling, eps 1e-3), double-Q targets over the
 * post-burn-in window and TF1 Adam(1e-4) without clipping.  Sequences are batch-major [B, S, ...].
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_r2d2 drl_r2d2;

typedef struct drl_r2d2_config {
  int32_t batch;              /* B sequences per step (config.json:94)                                   */
  int32_t seq_len;            /* S (config.json:95); BASELINE config 5 asks 80                           */
  int32_t burn_in;            /* loss window starts here (config.json:96), 0 <= burn_in <= S - 2         */
  int32_t height, width, channels; /* 84, 84, 1 (config.json:91) or 84, 84, 4                            */
  int32_t num_action;         /* A, 2..32                                                                */
  int32_t lstm_size;          /* 64 (config.json:93), 256 or 512; others -> DRL_ERR_INVALID. 256 and 512 run the
                                 recurrence on a thread-block cluster of lstm_size / 32 CTAs; the policy engine
                                 only syncs from a 64-wide learner                                       */
  float discount_factor;      /* agent/r2d2.py:62                                                        */
  float learning_rate;        /* 1e-4 (agent/r2d2.py:91)                                                 */
  int32_t device;
  int32_t num_slots;
  int32_t use_cuda_graph;
  int32_t math_mode;          /* 0 = default (2); 1 = FP32 FFMA; 2 = wgmma 3xTF32 for the large contractions */
  int32_t n_step;             /* 0 or 1 = the reference's one-step double-Q target (agent/r2d2.py:62-88).  n in
                                 [2, seq_len - burn_in - 1] = the R2D2 paper's n-step target: window t bootstraps from
                                 step t + k, k = min(n, seq_len - 1 - t), through the discounted rewards r[t..t+k-1]; a
                                 done inside the horizon cuts every later reward and the bootstrap (DESIGN.md section
                                 22).  Negative or larger values -> DRL_ERR_INVALID, before any device lookup. */
  int32_t priority_rule;      /* the per-sequence |td| of drl_r2d2_step / _wait / _td_error and of the device replay
                                 memory's priorities: 0 = |mean_t td| (agent/r2d2.py:154-157); 1 = the R2D2 paper's
                                 priority_eta max_t |td| + (1 - priority_eta) mean_t |td|.  Other values ->
                                 DRL_ERR_INVALID, before any device lookup.  The loss is the same under both rules. */
  float priority_eta;         /* read when priority_rule = 1 (the paper uses 0.9): finite and in [0, 1], otherwise
                                 DRL_ERR_INVALID, before any device lookup */
} drl_r2d2_config;

typedef struct drl_r2d2_out {
  float loss;        /* value_loss (agent/r2d2.py:90) */
  float grad_norm;   /* global gradient norm (diagnostic; the reference does not clip) */
  int64_t step;      /* updates applied so far */
} drl_r2d2_out;

int drl_r2d2_create(const drl_r2d2_config* cfg, drl_r2d2** out);
int drl_r2d2_destroy(drl_r2d2* h);
int drl_r2d2_param_count(const drl_r2d2* h, int64_t* n);   /* floats of ONE scope */
/* Flat float32 vector of scope `which` (0 = main, 1 = target) in TF layouts / TF variable-creation order: conv2d x3
 * (HWIO), dense x2 (action embedding), rnn/lstm_cell kernel [3136+256+L, 4L] (gate order i,j,f,o) + bias, dense 128,
 * dense A (value), dense 1 (mean). */
int drl_r2d2_set_params(drl_r2d2* h, int32_t which, const float* host_flat, int64_t n);
int drl_r2d2_get_params(drl_r2d2* h, int32_t which, float* host_flat, int64_t n);
int drl_r2d2_set_opt_state(drl_r2d2* h, const float* host_m, const float* host_v, int64_t n, int64_t step,
                           float beta1_power, float beta2_power);
int drl_r2d2_get_opt_state(drl_r2d2* h, float* host_m, float* host_v, int64_t n, int64_t* step,
                           float* beta1_power, float* beta2_power);
int drl_r2d2_get_grads(drl_r2d2* h, float* host_flat, int64_t n);
/* Agent.main_to_target (agent/r2d2.py:164-165, utils.py:27-32): target <- main. */
int drl_r2d2_main_to_target(drl_r2d2* h);
/* Feed of Agent.train (agent/r2d2.py:132-152): state u8 [B,S,H,W,C]; previous_action, action i32 [B,S]; h0, c0 f32
 * [B,L] (the reference feeds np.stack(h)[:, 0] of the stored [B,S,L] states); reward f32 [B,S]; done u8/bool [B,S];
 * weight f32 [B] or NULL (= ones). */
int drl_r2d2_stage(drl_r2d2* h, int32_t slot, const uint8_t* state, const int32_t* previous_action,
                   const int32_t* action, const float* h0, const float* c0, const float* reward, const uint8_t* done,
                   const float* weight);
/* sess.run([value_loss, target_value, state_action_value, train_op]) (agent/r2d2.py:134-152): both unrolls, TD
 * targets, loss, BPTT through all S steps of the main scope, Adam.  td_error (host [B], may be NULL) receives
 * |mean_t(target_value - state_action_value)| per sequence from BEFORE the update (agent/r2d2.py:154-157). */
int drl_r2d2_step(drl_r2d2* h, int32_t slot, drl_r2d2_out* out, float* td_error);
int drl_r2d2_step_async(drl_r2d2* h, int32_t slot);
int drl_r2d2_wait(drl_r2d2* h, drl_r2d2_out* out, float* td_error);
/* (new) Data-parallel halves, as drl_apex_forward_backward / _grad_bucket / _apply (value_loss is a batch mean,
 * agent/r2d2.py:90: grad_scale = 1 / world_size). */
int drl_r2d2_forward_backward(drl_r2d2* h, int32_t slot);
int drl_r2d2_grad_bucket(drl_r2d2* h, void** dev_ptr, int64_t* count);
int drl_r2d2_apply(drl_r2d2* h, float grad_scale);
/* Agent.get_td_error (agent/r2d2.py:97-130) for n <= batch sequences at once: td_error[i] = |mean(target - q)| of
 * sequence i (the reference calls it with one sequence). */
int drl_r2d2_td_error(drl_r2d2* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                      const int32_t* action, const float* h0, const float* c0, const float* reward,
                      const uint8_t* done, float* td_error);
/* Agent.get_action without the epsilon-greedy draw (agent/r2d2.py:171-191): one network step for n <= batch*seq_len
 * (state, previous_action, h, c) rows -> q_value [n,A], h' [n,L], c' [n,L]. */
int drl_r2d2_act(drl_r2d2* h, int32_t n, const uint8_t* state, const int32_t* previous_action, const float* h_in,
                 const float* c_in, float* q_value, float* h_out, float* c_out);
/* Parity taps of the most recent step / td_error call over its n sequences: main_q, target_q [n,S,A] (agent/r2d2.py:52),
 * target_value, state_action_value [n, S - burn_in - 1] (:81-88).  Any pointer may be NULL. */
int drl_r2d2_taps(drl_r2d2* h, float* main_q, float* target_q, float* target_value, float* state_action_value);
/* Debug/parity: named device buffer of the main scope (time-major rows m = t*n + b): a1 a2 a3 e1 emb q1 hout hin cin
 * gates dz dhout da3. */
int drl_r2d2_read_buffer(drl_r2d2* h, const char* name, float* host_dst, int64_t n);
int drl_r2d2_profile_step(drl_r2d2* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels,
                          int32_t* count);
int drl_r2d2_last_step_ms(drl_r2d2* h, float* ms);
int drl_r2d2_stream(drl_r2d2* h, void** stream);
int drl_r2d2_launches_per_step(const drl_r2d2* h, int32_t* n);
/* The recurrence's placement: CTAs per cluster (lstm_size / 32; 0 at lstm_size 64, which runs one CTA per sequence)
 * and how many clusters of the forward / BPTT kernel the device places at once (cudaOccupancyMaxActiveClusters at
 * create time; each launch uses at most that many, one per 8 (L = 256) or 4 (L = 512) sequences). */
int drl_r2d2_recurrence_clusters(const drl_r2d2* h, int32_t* cluster_size, int32_t* max_fwd, int32_t* max_bwd);

/* ------------------------------------------------------------------------------------------
 * R2D2 prioritized sequence replay memory on the device (DESIGN.md section 11): buffer_queue.Memory with one
 * stored-state sequence per record in HBM (state u8 [S,84,84,C]; previous_action, action i32 [S]; reward f32 [S]; done
 * u8 [S]; h0, c0 f32 [L], step 0 of the stored states, the only step the learner reads; zero-initialised), the float64
 * sum tree on the device, and the learner loop of train_r2d2.py:87-165 -- ingest, sample, minibatch gather, step,
 * priority update -- as kernels on the learner's compute stream.  The sum tree, its constants and arithmetic and the
 * sample / update / last_sample / total / size / beta calls behave as drl_apex_replay_*'s.  The memory outlives any
 * learner: every call that uses one takes a drl_r2d2* on the memory's device with the memory's seq_len, channels,
 * num_action and lstm_size L, and orders itself after the memory's previous work on whichever stream that ran.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_r2d2_replay drl_r2d2_replay;
/* capacity in [2, 2^31], seq_len >= 2, channels 1 or 4, num_action in [2, 32]; lstm_size L = 64.  Device memory per
 * sequence: S * (7,056 C + 13) + 8 L bytes: 106,547 B at S = 15, C = 1, L = 64 (10.7 GB at the reference's capacity
 * 1e5), 424,067 B at C = 4 (42.4 GB). */
int drl_r2d2_replay_create(int32_t device, int64_t capacity, int32_t seq_len, int32_t channels, int32_t num_action,
                           drl_r2d2_replay** out);
/* drl_r2d2_replay_create for lstm_size L in {64, 256, 512} (others -> DRL_ERR_INVALID). */
int drl_r2d2_replay_create_lstm(int32_t device, int64_t capacity, int32_t seq_len, int32_t channels, int32_t num_action,
                                int32_t lstm_size, drl_r2d2_replay** out);
int drl_r2d2_replay_destroy(drl_r2d2_replay* r);
/* Memory.add for n sequences in order at the write cursor (wrapping); the arguments are drl_r2d2_td_error's (h0, c0
 * [n, L]).  error == NULL: the priorities are the learner's |td| of these sequences (agent/r2d2.py:97-130, all n in
 * one pass), computed on the device and never copied to the host; then 1 <= n <= the learner's batch.  Otherwise
 * error [n] are the caller's and learner may be NULL.  Every previous_action and action must be in [0, num_action).
 * Does not wait for the learner's compute stream. */
int drl_r2d2_replay_add(drl_r2d2_replay* r, drl_r2d2* learner, int32_t n, const uint8_t* state,
                        const int32_t* previous_action, const int32_t* action, const float* h0, const float* c0,
                        const float* reward, const uint8_t* done, const double* error);
/* Memory.sample(B) with the caller's uniforms u01 [B] (B = the learner's batch) -> gather into staging slot `slot` ->
 * the learner's step on that slot -> Memory.update of the sampled leaves with the step's |td|.  Asynchronous:
 * drl_r2d2_wait returns the loss and the priorities once the update has run.  DRL_ERR_STATE on an empty memory. */
/* drl_r2d2_replay_add of the oldest full batch of a device R2D2 queue (train_r2d2.py:97-120 without a host copy): pops it
 * without holding the memory's or the learner's lock, blocking while fewer than batch sequences are queued
 * (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with nothing changed otherwise), then, on the learner's compute stream, the
 * learner's |td| of the batch read from the queue slot, the store and the priority update; the slot goes back to the
 * producers after them, also when enqueueing fails.  The queue's seq_len, channels, num_action and device must be the
 * memory's, the memory's lstm_size the queue's 64, and the queue's batch at most the learner's (DRL_ERR_INVALID).  Does not wait for the learner's compute stream. */
int drl_r2d2_replay_add_from_queue(drl_r2d2_replay* r, drl_r2d2* learner, drl_r2d2_queue* queue, int32_t timeout_ms);
int drl_r2d2_replay_step_async(drl_r2d2_replay* r, drl_r2d2* learner, int32_t slot, const double* u01);
/* As drl_apex_replay_sample / _update / _last_sample. */
int drl_r2d2_replay_sample(drl_r2d2_replay* r, int32_t n, const double* u01, int64_t* tree_index,
                           int64_t* data_index, double* priority, double* is_weight);
int drl_r2d2_replay_update(drl_r2d2_replay* r, int32_t n, const int64_t* tree_index, const double* error);
int drl_r2d2_replay_last_sample(drl_r2d2_replay* r, int64_t* tree_index, double* priority, double* is_weight);
/* Rows [data_index, data_index + n) of the storage (h0, c0 [n, 64]); any pointer may be NULL. */
int drl_r2d2_replay_read(drl_r2d2_replay* r, int64_t data_index, int32_t n, uint8_t* state, int32_t* previous_action,
                         int32_t* action, float* h0, float* c0, float* reward, uint8_t* done);
int drl_r2d2_replay_total(drl_r2d2_replay* r, double* total);      /* SumTree.total */
int drl_r2d2_replay_size(drl_r2d2_replay* r, int64_t* n_entries);  /* SumTree.n_entries */
int drl_r2d2_replay_beta(drl_r2d2_replay* r, double* beta);

/* ------------------------------------------------------------------------------------------
 * A3C learner: replaces a3c.Agent's learner graph (agent/a3c.py:11-78) over model/actor_critic.py:3-56 (the same body
 * as the Ape-X network: attention_CNN || action embedding -> concat 3392 -> actor [256,256,A + softmax] and critic
 * [256,256,1]) and optimizer/a2c.py:3-26, with TF1 Adam + polynomial decay + global-norm clipping.  network(s, prev_a)
 * and network(s', a) run as ONE forward over 2B rows; next_value is stop_gradient, so only the first B rows are
 * differentiated.  The handle is the Ape-X handle type in A3C mode.
 * ------------------------------------------------------------------------------------------ */
typedef struct drl_apex drl_a3c;

typedef struct drl_a3c_config {
  int32_t batch;              /* transitions per step: trajectory (config.json:36) -- the learner trains on one unroll */
  int32_t height, width, channels; /* 84,84,4                                                           */
  int32_t num_action;
  float discount_factor;      /* agent/a3c.py:45                                                        */
  float start_learning_rate;  /* agent/a3c.py:76                                                        */
  float end_learning_rate;
  double learning_frame;
  float baseline_loss_coef;   /* agent/a3c.py:73                                                        */
  float entropy_coef;
  float gradient_clip_norm;   /* agent/a3c.py:79                                                        */
  int32_t reward_clipping;    /* DRL_REWARD_ABS_ONE / DRL_REWARD_SOFT_ASYMMETRIC (agent/a3c.py:38-43)    */
  int32_t device;
  int32_t num_slots;
  int32_t use_cuda_graph;
  int32_t math_mode;
} drl_a3c_config;

typedef struct drl_a3c_out {
  float pi_loss;        /* -mean(advantage * pi(a))           (optimizer/a2c.py:17-26) */
  float baseline_loss;  /* mean((r + gamma V(s') - V(s))^2)    (optimizer/a2c.py:9-15)  */
  float entropy;        /* -mean(sum_a -pi log pi)             (optimizer/a2c.py:3-7)   */
  float learning_rate;
  float grad_norm;
  int64_t step;
} drl_a3c_out;

int drl_a3c_create(const drl_a3c_config* cfg, drl_a3c** out);
int drl_a3c_destroy(drl_a3c* h);
int drl_a3c_param_count(const drl_a3c* h, int64_t* n);
/* Flat float32 vector, TF variable order of scope {model}/a3c: conv2d x3, dense x2 (embedding), dense x3 (actor),
 * dense x3 (critic). */
int drl_a3c_set_params(drl_a3c* h, const float* host_flat, int64_t n);
int drl_a3c_get_params(drl_a3c* h, float* host_flat, int64_t n);
int drl_a3c_set_opt_state(drl_a3c* h, const float* host_m, const float* host_v, int64_t n, int64_t step,
                          float beta1_power, float beta2_power);
int drl_a3c_get_opt_state(drl_a3c* h, float* host_m, float* host_v, int64_t n, int64_t* step, float* beta1_power,
                          float* beta2_power);
int drl_a3c_get_grads(drl_a3c* h, float* host_flat, int64_t n);
/* Feed of Agent.train (agent/a3c.py:85-103): state, next_state u8 [B,H,W,C]; previous_action, action i32 [B] (the
 * reference feeds `action` as the next step's previous action, :99); reward f32 [B]; done u8/bool [B]. */
int drl_a3c_stage(drl_a3c* h, int32_t slot, const uint8_t* state, const uint8_t* next_state,
                  const int32_t* previous_action, const int32_t* action, const float* reward, const uint8_t* done);
/* sess.run([pi_loss, baseline_loss, entropy, learning_rate, train_op]) (agent/a3c.py:89-103). */
int drl_a3c_step(drl_a3c* h, int32_t slot, drl_a3c_out* out);
/* drl_a3c_stage of the oldest record of a device A3C queue (train_a3c.py's learner loop without a host copy): pops it
 * without holding the learner's lock, blocking while the queue is empty (timeout_ms < 0: forever; DRL_ERR_TIMEOUT with
 * nothing changed otherwise), then, on the copy stream after the slot's last reader and the record's commit, copies it
 * device to device into `slot` (weights 1, as drl_a3c_stage) and records the slot's staged event; the queue slot goes
 * back to the producers after the copies, also when enqueueing fails.  The learner must be an A3C handle on the queue's
 * device with batch = the queue's trajectory and the queue's num_action (DRL_ERR_INVALID). */
int drl_a3c_stage_from_queue(drl_a3c* h, int32_t slot, drl_a3c_queue* queue, int32_t timeout_ms);
int drl_a3c_step_async(drl_a3c* h, int32_t slot);
int drl_a3c_wait(drl_a3c* h, drl_a3c_out* out);
/* (new) Data-parallel halves (all three A2C losses are batch means: grad_scale = 1 / world_size). */
int drl_a3c_forward_backward(drl_a3c* h, int32_t slot);
int drl_a3c_grad_bucket(drl_a3c* h, void** dev_ptr, int64_t* count);
int drl_a3c_apply(drl_a3c* h, float grad_scale);
/* Agent.get_policy_and_action without the sampling (agent/a3c.py:109-119): policy [n,A] and value [n], n <= 2*batch. */
int drl_a3c_act(drl_a3c* h, int32_t n, const uint8_t* state, const int32_t* previous_action, float* policy,
                float* value);
/* Parity taps of the most recent step: policy [B,A], value [B], next_value [B], advantage [B]. */
int drl_a3c_taps(drl_a3c* h, float* policy, float* value, float* next_value, float* advantage);
int drl_a3c_read_buffer(drl_a3c* h, const char* name, float* host_dst, int64_t n);
int drl_a3c_profile_step(drl_a3c* h, int32_t slot, char* names, int64_t names_len, float* ms, int32_t max_kernels,
                         int32_t* count);
int drl_a3c_stream(drl_a3c* h, void** stream);
int drl_a3c_launches_per_step(const drl_a3c* h, int32_t* n);

#ifdef __cplusplus
}
#endif
#endif /* DRL_B200_H_ */
