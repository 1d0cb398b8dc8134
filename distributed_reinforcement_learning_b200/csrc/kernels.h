// kernels.h -- internal interface between the learner orchestration (learner_core.cu with learner.cu; adam_learner.cu with apex.cu and
// r2d2.cu) and the kernel launchers (layers.cu, elementwise.cu, vtrace.cu, optimizer.cu).  Not part of the C-ABI.
#pragma once
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: no link dependency, a no-op unless a profiler injects itself

#include "common.cuh"

namespace drl {

// an NVTX range over a host-side phase (the learners' step phases, the policy engines' calls); SURVEY.md section 5:
// the reference has no tracing at all
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// Offsets (in floats) of each tensor inside the padded flat parameter / gradient / slot vectors of one network.
// Order = TF1 variable-creation order (SURVEY.md App. A.6); every bias directly follows its
// kernel (kernel sizes are multiples of 4) and is padded up to a multiple of 4 floats so that all
// kernels start 16-byte aligned.  [w ; b] therefore forms one contiguous [(K+1), N] matrix, which
// is what the weight-gradient GEMMs write (bias gradient = column sum of dY in row K).
// The C-ABI exchanges the packed (TF-flat) vector; the device holds the padded one.
struct FlatLayout {
  static constexpr int kMaxTensors = 24;
  int num_tensors = 0;
  int64_t padded_total = 0;   // floats in the padded vector (multiple of 4)
  int64_t packed_total = 0;   // floats in the TF-flat (API) vector
  int64_t packed_off[kMaxTensors], padded_off[kMaxTensors], count[kMaxTensors];
  // offsets of the tensors of sizes[] (kernel, bias, kernel, bias, ...); *named[i] receives padded_off[i]
  template <int N>
  void set(const int64_t (&sizes)[N], int64_t* const (&named)[N]) {
    static_assert(N <= kMaxTensors, "too many tensors");
    set(N, sizes, named);
  }
  void set(int n, const int64_t* sizes, int64_t* const* named);
};

// The tensors every network here starts with, in this order: the attention_CNN (conv1, conv2, conv3) and the action
// embedding (emb1, emb2).  The IMPALA, Ape-X / A3C and R2D2 layouts derive from it.
struct TrunkLayout : FlatLayout {
  int A;
  int C = Geo::IC;   // input channels (R2D2: 1 or 4)
  int64_t conv1_w, conv1_b, conv2_w, conv2_b, conv3_w, conv3_b;
  int64_t emb1_w, emb1_b, emb2_w, emb2_b;
};

struct ParamLayout : TrunkLayout {   // IMPALA network
  int64_t lstm_w, lstm_b;
  int64_t actor1_w, actor1_b, actor2_w, actor2_b, actor3_w, actor3_b;
  int64_t critic1_w, critic1_b, critic2_w, critic2_b, critic3_w, critic3_b;
  void init(int num_action);
};

// packed (API) <-> padded (device) copies through the pinned staging buffer `h_flat` (padded_total floats) on stream
// `s`; both return once the copy is complete.  upload fills the padding with pad_value.
int upload_flat(cudaStream_t s, float* h_flat, const FlatLayout& pl, float* dev_padded, const float* host_packed,
                float pad_value);
int download_flat(cudaStream_t s, float* h_flat, const FlatLayout& pl, const float* dev_padded, float* host_packed);

// cudaMalloc + memset of count elements plus 256 bytes of slack (kernels may read a vector's tail past its end);
// the handle's `allocs` list owns the memory
template <class H, class T>
int dev_alloc(H* h, T** p, size_t count, int fill_byte = 0) {
  void* q = nullptr;
  DRL_CUDA_CHECK(cudaMalloc(&q, count * sizeof(T) + 256));
  DRL_CUDA_CHECK(cudaMemset(q, fill_byte, count * sizeof(T) + 256));
  h->allocs.push_back(q);
  *p = static_cast<T*>(q);
  return DRL_OK;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Captures what enqueue() (-> DRL_OK or an error code) issues on stream s into an instantiated graph.  A failing
// enqueue or capture leaves *exec untouched.
template <class F>
int capture_graph(cudaStream_t s, F&& enqueue, cudaGraphExec_t* exec) {
  cudaGraph_t g = nullptr;
  DRL_CUDA_CHECK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
  const int r = enqueue();
  const cudaError_t e = cudaStreamEndCapture(s, &g);
  if (r != DRL_OK) { if (g) cudaGraphDestroy(g); return r; }
  if (e != cudaSuccess) { set_error("graph capture failed: %s", cudaGetErrorString(e)); return DRL_ERR_CUDA; }
  DRL_CUDA_CHECK(cudaGraphInstantiate(exec, g, 0));
  cudaGraphDestroy(g);
  return DRL_OK;
}

struct Inputs {          // one device staging slot, caller's batch-major layout
  const uint8_t* frames; // [B,T,84,84,4]
  const float* reward;   // [B,T]
  const int32_t* action; // [B,T]
  const uint8_t* done;   // [B,T]
  const float* mu;       // [B,T,A]
  const int32_t* pa;     // [B,T]
  const float* h0;       // [B,T,256]
  const float* c0;       // [B,T,256]
};

// The trunk's forward activations over M rows and its backward workspace over Mb rows (the rows that receive gradient),
// the bases of every learner's activation and workspace structs.
struct TrunkActs {
  float* a1;             // [M,20,20,32]
  float* a2;             // [M,9,9,64]
  float* a3;             // [M,3136]
  float* e1;             // [A,256]  relu(emb1)
  float* table;          // [A,256]  action-embedding table
  // math mode 5: 16-bit [hi | lo] planes of a1 / a2 (Plane16, split16.cuh), written beside them by conv1_fwd / conv2_fwd
  // and read by conv2_fwd / conv3_fwd; 2 x 2 bytes per element, nullptr where not kept
  uint16_t* a1p = nullptr;
  uint16_t* a2p = nullptr;
};
struct TrunkBwd {
  float* da3;            // [Mb,3136]
  float* du;             // [Mb,256]
  float* dpre2;          // [A,256]
  float* dpre1;          // [A,256]
  float* da2;            // [Mb,9,9,64]
  float* da1;            // [Mb,20,20,32]
  float* wg_part;        // split-K partial slabs for the conv3/conv2 weight gradients (side stream) + emb scratch
  float* wg_part2;       // split-K partial slabs for the conv1 weight gradient (main stream)
  float* dcol = nullptr; // [Mb*81, 512] (conv2) / [Mb*49, 576] (conv3): per-output-pixel tap gradients before col2im
                         // (math modes 2 and 3; math mode 5 computes the conv data gradients without it)
  // math mode 5: 16-bit planes of da3 / da2, written beside them by lstm_dgrad / conv3_dgrad and read by conv3_dgrad /
  // conv2_dgrad (as TrunkActs::a1p)
  uint16_t* da3p = nullptr;
  uint16_t* da2p = nullptr;
};
// floats of wg_part / wg_part2 for Mb rows of C-channel frames: the largest split-K slab set of the conv weight gradients
// in any math mode, at least the scratch of emb_backward
size_t trunk_partial_floats(int Mb, int C);
template <class H>
int alloc_trunk_acts(H* h, TrunkActs& a, size_t M, size_t A, bool planes = false) {
  DRL_TRY(dev_alloc(h, &a.a1, M * 400 * 32));
  DRL_TRY(dev_alloc(h, &a.a2, M * 81 * 64));
  DRL_TRY(dev_alloc(h, &a.a3, M * Geo::FLAT));
  DRL_TRY(dev_alloc(h, &a.e1, A * Geo::EMB));
  DRL_TRY(dev_alloc(h, &a.table, A * Geo::EMB));
  if (planes) {
    DRL_TRY(dev_alloc(h, &a.a1p, 2 * M * 400 * 32));
    DRL_TRY(dev_alloc(h, &a.a2p, 2 * M * 81 * 64));
  }
  return DRL_OK;
}
template <class H>
int alloc_trunk_bwd(H* h, TrunkBwd& b, size_t Mb, size_t A, int C, bool dcol, bool planes = false) {
  DRL_TRY(dev_alloc(h, &b.da3, Mb * Geo::FLAT));
  DRL_TRY(dev_alloc(h, &b.du, Mb * Geo::EMB));
  DRL_TRY(dev_alloc(h, &b.dpre2, A * Geo::EMB));
  DRL_TRY(dev_alloc(h, &b.dpre1, A * Geo::EMB));
  DRL_TRY(dev_alloc(h, &b.da2, Mb * 81 * 64));
  DRL_TRY(dev_alloc(h, &b.da1, Mb * 400 * 32));
  const size_t wg = trunk_partial_floats((int)Mb, C);
  DRL_TRY(dev_alloc(h, &b.wg_part, wg));
  DRL_TRY(dev_alloc(h, &b.wg_part2, wg));
  if (dcol) DRL_TRY(dev_alloc(h, &b.dcol, Mb * 81 * 512));
  if (planes) {
    DRL_TRY(dev_alloc(h, &b.da3p, 2 * Mb * Geo::FLAT));
    DRL_TRY(dev_alloc(h, &b.da2p, 2 * Mb * 81 * 64));
  }
  return DRL_OK;
}

struct Acts : TrunkActs { // forward activations, time-major rows m = t*B + b, M = B*T rows
  float* zpart;          // [SPLITS][M,1024] LSTM pre-activation partial sums
  float* gates;          // [M,4,256] sigmoid(i), tanh(j), sigmoid(f+1), sigmoid(o)
  float* c1;             // [M,256]
  float* tc1;            // [M,256] tanh(c1)
  float* h1;             // [M,256]
  float* hid1;           // [2][M,256] actor/critic hidden 1
  float* hid2;           // [2][M,256] actor/critic hidden 2
  float* logits;         // [M,A]
  float* policy;         // [M,A]
  float* value;          // [M]
  // math mode 5, bulk-fed lstm_wgrad (gemm_bulk16.cuh): x^T = [a3|emb|h0]^T as a 16-bit operand image
  uint8_t* img_xt = nullptr;   // x^T : rows = features (3648) x K = Mb rows -- A operand of lstm_wgrad
  // recurrent mode only (Recurrence): the summed input half of the pre-activation and the state each step read
  float* zx = nullptr;         // [M,1024] [a3 | emb] W[:3392]
  float* hin = nullptr;        // [M,256]
  float* cin = nullptr;        // [M,256]
};

struct Bwd : TrunkBwd {  // backward workspace, Mb = B*(T-2) rows
  float* dlogits;        // [Mb,32] (columns >= A stay zero)
  float* dv;             // [Mb,32] (column 0 = dL/dV, others stay zero)
  float* dhid2;          // [2][Mb,256]
  float* dhid1;          // [2][Mb,256]
  float* dh_part;        // [2][Mb,256] actor and critic contributions to dL/dh1
  float* dz;             // [Mb,1024]
  uint8_t* img_dzt = nullptr;  // dz^T : rows n (1024) x K = Mb rows  -- B operand of the bulk-fed lstm_wgrad (see Acts::img_xt)
  size_t wg_part_floats; // floats of wg_part / wg_part2 (checked by the conv1 weight gradient of math mode 5)
  float* emb_scratch = nullptr;   // own scratch of emb_backward (16 * 32 * 256 floats): lets it run on the second side lane
                                  // beside the conv weight gradients; nullptr: it borrows wg_part on `side`
};

struct VtraceOut {       // parity taps, batch-major [B, T-2]
  float *vs, *clipped_rho, *vs_plus_1, *pg_adv;
  float* loss_partials;  // [nblk,3]
  unsigned int* ticket;  // last-block counter
  float* loss_sums;      // [4] pi, baseline, entropy, (pad) -- tail of the gradient bucket
};

constexpr int kLstmSplits = 8;   // slabs allocated for the LSTM split-K partial sums (4 or 7 are used)

// math_mode 0 in drl_learner_config resolves to this (1 = FP32 FFMA, 2 = wgmma 3xTF32)
#ifndef DRL_DEFAULT_MATH_MODE
#define DRL_DEFAULT_MATH_MODE 2          // Ape-X / A3C / R2D2 handles
#endif
#ifndef DRL_DEFAULT_MATH_MODE_IMPALA
#define DRL_DEFAULT_MATH_MODE_IMPALA 5   // IMPALA handle: wgmma with 16-bit split operands (gemm_umma16.cuh)
#endif

// Per-kernel device timing (learner_core.cu): when a profile run is active, prof_mark records a CUDA event
// on the launching stream before each named launch; otherwise it is a no-op.
void prof_mark(cudaStream_t s, const char* name);
// profile run bracket (shared by the IMPALA and the Ape-X learner): prof_begin arms prof_mark; prof_end synchronises
// `s`, converts the recorded events into per-launch times (names joined by '\n') and disarms it.
void prof_begin();
int prof_end(cudaStream_t s, int rc, char* names, int64_t names_len, float* ms, int32_t max_kernels, int32_t* count);

// Pre-split (hi/lo tf32), pre-tiled, pre-swizzled global copies of the weights that serve as B operands of the
// tensor-core GEMMs (gemm_umma.cuh: PretiledB / retile_b_kernel); refreshed after every parameter update.
struct WeightImages {
  static constexpr int kCount = 7;
  // 0 conv1 fwd (no reader: every conv1 kernel reads the fp32 weights; kept because the Ape-X / R2D2 handles size their
  // images with the same weight_image_sizes), 1 conv2 fwd, 2 conv3 fwd, 3 lstm fwd, 4 lstm dgrad, 5 conv3 dCol, 6 conv2 dCol
  uint8_t* img[kCount];
};
void weight_image_sizes(size_t (&bytes)[WeightImages::kCount]);
int net_retile(cudaStream_t s_conv, cudaStream_t s_rest, const ParamLayout& pl, const float* params,
               const WeightImages& wi);

// ---- layers.cu ----------------------------------------------------------------------------
// main = critical path; side = kernels off the critical path (fork/join through ev[]); par = false runs
// everything on main (used by the per-kernel profile so that event times are per-kernel).
struct Streams {
  cudaStream_t main, side;
  cudaEvent_t ev[8];
  bool par;
  // optional second side lane (IMPALA handle): the four small, latency-bound head weight gradients run here so that they
  // do not sit in front of lstm_wgrad / the conv weight gradients on `side` (tools/timeline.py, profiles/r02_timeline_*).
  // nullptr: everything stays on `side`.
  cudaStream_t side2 = nullptr;
  cudaEvent_t ev2[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_lstm_grads = nullptr;   // backward: recorded on the side stream once the head and LSTM weight gradients
                                         // are in the bucket (the early part of the peer exchange waits for it)
};
// The IMPALA learner's recurrent mode (drl_learner_config.recurrent = 1): the LSTM runs through the T steps of each
// trajectory on the cluster kernels of r2d2_cluster.cuh (RESTART variant), which the device places this many clusters of
// at once.  Zero clusters: the stored-state mode, one LSTM step per row from the recorded (h, c).
struct Recurrence {
  int clusters_fwd = 0, clusters_bwd = 0;
  bool on() const { return clusters_fwd > 0; }
};
// Create-time set-up of the recurrent mode's kernels (dynamic shared memory, occupancy); DRL_ERR_CUDA if no cluster fits
int impala_recurrence_setup(Recurrence* rec);
// mode: 1 = FP32-FFMA gather-GEMM, 2 = wgmma 3xTF32 gather-GEMM for the large contractions
int net_forward(const Streams& st, const ParamLayout& pl, const float* params, const WeightImages& wi, const Inputs& in,
                const Acts& act, int B, int T, int mode, bool retile, const Recurrence& rec);
int net_backward(const Streams& st, const ParamLayout& pl, const float* params, const WeightImages& wi, float* grads,
                 const Inputs& in, const Acts& act, const Bwd& bwd, int B, int T, int mode, const Recurrence& rec);
// bytes of the operand images of the bulk-fed lstm_wgrad: which = 1 x^T (K = Mb), 3 dz^T (K = Mb)
size_t lstm_image_bytes(int which, int M, int Mb);
int forward_launch_count();
int backward_launch_count();
// the IMPALA policy engine's convolutions (policy.cu): the math-mode-5 conv1 / conv2 / conv3 forward of net_forward over
// n single frames on one stream, and the build of its conv2 / conv3 weight images (WeightImages slots 1 and 2 sizes);
// a1p / a2p: the 16-bit planes of a1 / a2 (TrunkActs::a1p) for n rows
int conv_images16(cudaStream_t s, const ParamLayout& pl, const float* params, uint8_t* img_conv2, uint8_t* img_conv3);
int conv_forward16(cudaStream_t s, const ParamLayout& pl, const float* params, const uint8_t* img_conv2,
                   const uint8_t* img_conv3, const uint8_t* frames, int n, float* a1, float* a2, float* a3,
                   uint16_t* a1p, uint16_t* a2p);
// the Ape-X / A3C and R2D2 policy engines' convolutions (apex_policy.cu, r2d2_policy.cu; defined in r2d2.cu, whose
// learner instantiates both channel counts): the math-mode-2 conv_forward_tf32 of layer_defs.cuh over n single frames
// of pl.C channels, and conv_images_tf32
int policy_conv_forward_tf32(cudaStream_t s, const TrunkLayout& pl, const float* params, const uint8_t* img_conv2,
                             const uint8_t* img_conv3, const uint8_t* frames, int n, float* a1, float* a2, float* a3);
int policy_conv_images_tf32(cudaStream_t s, const TrunkLayout& pl, const float* params, uint8_t* img_conv2,
                            uint8_t* img_conv3);

// ---- policy.cu: the IMPALA policy engine's act on device-resident inputs (policy_server.cu) ------------------------
struct PolicyCore;
PolicyCore* policy_core_of(drl_policy* h);
// the rows of an n-row act inside the engine's device input block
struct PolicyInRows {
  uint8_t* frames;   // [n][84*84*4]
  int32_t* pa;       // [n]
  float* h0;         // [n][256]
  float* c0;         // [n][256]
  double* uniform;   // [n]
};
// where the act's head writes: policy [n][A], h1 / c1 [n][256], action [n]
struct PolicyOutRows {
  float* policy;
  float* h1;
  float* c1;
  int32_t* action;
};
PolicyInRows policy_input_rows(drl_policy* h, int n);
// the engine's act kernels of n rows (drl_policy_act without the upload of its input block) on the engine's stream,
// reading the rows of policy_input_rows(h, n) and writing `out`; the caller holds the engine's lock
int policy_enqueue_forward(drl_policy* h, int n, const PolicyOutRows& out);

// ---- r2d2_policy.cu: the R2D2 policy engine's act on device-resident inputs (r2d2_policy_server.cu) ---------------
PolicyCore* r2d2_policy_core_of(drl_r2d2_policy* h);
int r2d2_policy_channels(const drl_r2d2_policy* h);   // C of the engine's 84x84xC frames
// the rows of an n-row act inside the engine's device input block
struct R2PolicyInRows {
  uint8_t* frames;   // [n][84*84*C]
  int32_t* pa;       // [n]
  float* h0;         // [n][64]
  float* c0;         // [n][64]
  int32_t* explore;  // [n]: -1 greedy, otherwise the action (in [0, A): the head indexes q with it)
};
// where the act's head writes: q [n][A], h1 / c1 [n][64], action [n], q_action [n]
struct R2PolicyOutRows {
  float* q;
  float* h1;
  float* c1;
  int32_t* action;
  float* q_action;
};
R2PolicyInRows r2d2_policy_input_rows(drl_r2d2_policy* h, int n);
// the engine's act kernels of n rows (drl_r2d2_policy_act without the upload of its input block: conv stack,
// policy_lstm_fwd and r2d2_policy_head_kernel) on the engine's stream, reading the rows of r2d2_policy_input_rows(h, n)
// and writing `out`; the caller holds the engine's lock
int r2d2_policy_enqueue_forward(drl_r2d2_policy* h, int n, const R2PolicyOutRows& out);

// ---- apex_policy.cu: the Ape-X / A3C policy engine's act on device-resident inputs (a3c_policy_server.cu) ---------
PolicyCore* apex_policy_core_of(drl_apex_policy* h);
int apex_policy_algo(const drl_apex_policy* h);   // 0 = Ape-X, 1 = A3C
// the rows of an n-row act inside the engine's device input block
struct ApexPolicyInRows {
  uint8_t* frames;   // [n][84*84*4]
  int32_t* pa;       // [n]
  double* uniform;   // [n]: A3C's uniform draws (the Ape-X engine reads the same bytes as i32 explore actions)
};
// where the act's head writes: q or policy [n][A], action [n], q[action] or policy[action] [n]
struct ApexPolicyOutRows {
  float* out;
  int32_t* action;
  float* out_action;
};
ApexPolicyInRows apex_policy_input_rows(drl_apex_policy* h, int n);
// the engine's act kernels of n rows (drl_apex_policy_act / drl_a3c_policy_act without the upload of the input block:
// conv stack, skinny_splitk_fwd and apex_policy_head_kernel) on the engine's stream, reading the rows of
// apex_policy_input_rows(h, n) and writing `out`; the caller holds the engine's lock
int apex_policy_enqueue_forward(drl_apex_policy* h, int n, const ApexPolicyOutRows& out);

// ---- learner.cu: parameter snapshot for the policy engine (drl_policy_sync_from_learner) ---------------------------
// learner_params_snapshot (learner_core.cuh) of an IMPALA learner whose network has num_action actions:
// DRL_ERR_INVALID for a learner with another num_action, DRL_ERR_STATE for a learner in the failed state.
int impala_params_snapshot(drl_learner* h, int device, int num_action, cudaStream_t dst_stream, float* dst,
                           cudaEvent_t ev_ready, cudaEvent_t ev_copied);

// ---- elementwise.cu -----------------------------------------------------------------------
int emb_forward(cudaStream_t s, const float* w1, const float* b1, const float* w2, const float* b2, float* e1,
                float* table, int A);
int lstm_gates_forward(cudaStream_t s, const float* zpart, int nsplit, const float* bias, const float* c0,
                       float* gates, float* c1, float* tc1, float* h1, int M, int B, int T);
int heads_out_forward(cudaStream_t s, const float* hid2_actor, const float* hid2_critic, const float* w5,
                      const float* b5, const float* w8, const float* b8, float* logits, float* policy,
                      float* value, int M, int A);
int heads_out_backward(cudaStream_t s, const float* dlogits, const float* dv, const float* w5, const float* w8,
                       const float* hid2_actor, const float* hid2_critic, float* dhid2_actor, float* dhid2_critic,
                       int Mb, int A);
int lstm_gates_backward(cudaStream_t s, const float* dh_part, size_t part_stride, const float* gates,
                        const float* tc1, const float* c0, float* dz, int Mb, int B, int T);
int emb_backward(cudaStream_t s, const float* du, const int32_t* pa, const float* e1, const float* table,
                 const float* w2, float* dpre2, float* dpre1, float* g_w1, float* g_b1, float* g_w2, float* g_b2,
                 float* scratch, int Mb, int B, int T, int A);
int splitk_reduce(cudaStream_t s, const float* part, size_t slab, int nsplit, float* out, size_t n);
// second half of the "dCol" form of the conv data gradients (gather of <= 9 / 4 taps + ReLU mask)
int col2im_conv3(cudaStream_t s, const float* dcol, const float* a2, float* da2, int nimg);
int col2im_conv2(cudaStream_t s, const float* dcol, const float* a1, float* da1, int nimg);

// ---- vtrace.cu ----------------------------------------------------------------------------
struct VtraceCfg {
  float discount, baseline_coef, entropy_coef;
  int reward_clipping;
};
int vtrace_losses(cudaStream_t s, const VtraceCfg& cfg, const float* policy, const float* value, const Inputs& in,
                  const VtraceOut& out, float* dlogits, float* dv, int B, int T, int A);

// ---- optimizer.cu -------------------------------------------------------------------------
struct OptState {
  float* params; float* ms; float* grads;   // padded flat vectors
  int64_t n;                                 // padded_total (multiple of 4)
  float* norm_partials; int nblk;            // partial sums of squares; grid size of the two optimizer kernels
  int npart;                                 // how many partials the update kernel sums (nblk, or world * nblk_r)
  // peer exchange (peer.cu): the update kernel first waits for the peers' barrier-1 flags (null: single replica)
  const uint32_t* wait_flags; const uint32_t* wait_epoch; int wait_world;
  uint32_t* wait_err; uint32_t* wait_err_host; unsigned long long wait_timeout_ns;   // peer_sync.cuh::PeerErr
  int wait_parts;                            // exchange instances to wait for
  long long* step;                           // device global_step
  float* lr_cur;                             // device scalar
  float* out;                                // device [8]: pi, baseline, entropy, lr, grad_norm, total, step_lo, step_hi
  const float* loss_sums;                    // bucket tail
  float start_lr, end_lr; double learning_frame;
  float clip_norm, baseline_coef, entropy_coef;
};
int optimizer_apply(cudaStream_t s, const OptState& o);
int optimizer_update_only(cudaStream_t s, const OptState& o);   // clip + RMSProp from already reduced partials

// ---- adam_learner.cu: TF1 Adam (the Ape-X / A3C and the R2D2 learner) -------------------------------------------
// clip_norm <= 0: no clipping (optimizer.minimize, agent/r2d2.py:92); start_lr == end_lr: constant learning rate
struct AdamState {
  float* params; float* m; float* v; const float* grads; int64_t n;
  float* norm_partials; int nblk;
  long long* step; float* lr_cur; float* alpha; float* b1p; float* b2p;
  float* out;               // [8] mapped pinned: loss, lr, grad_norm, -, -, -, step_lo, step_hi
  const float* loss;
  float start_lr, end_lr; double learning_frame; float clip_norm;
  float grad_scale;         // data parallel: the bucket holds the SUM over ranks of per-rank MEAN-loss gradients -> 1/world
                            // (1 for a single replica); applied to the gradient, its norm and the logged losses
};
int adam_step(cudaStream_t s, const AdamState& o);   // 2 launches: partial norms + scalars, then the update

// ---- peer.cu: gradient exchange over NVLink peer memory (CUDA IPC), fused with the norm ------------------------
constexpr int kMaxPeers = 16;
constexpr int kPeerParts = 2;      // exchange instances per step: part 0 = [lstm .. end) of the bucket (96 % of the bytes, complete when
                                   // the LSTM weight gradient is, ~230 us before the backward pass ends) on its own stream with a small
                                   // grid; part 1 = [conv1 .. emb2] after the backward pass (see DESIGN.md section 5)
struct PeerTable {                 // device pointers into every rank's buffers (index = rank; own entries are local)
  float* bucket[kMaxPeers];        // [padded grads | 4 loss sums]
  float* reduced[kMaxPeers];       // same shape: the summed bucket, delivered by the owners of the slices
  float* partials[kMaxPeers];      // [world * nblk_r] partial squared norms
  uint32_t* flags[kMaxPeers];      // [2 * kPeerParts][kMaxPeers] barrier epochs (phase = 2 * part + {ready, delivered})
  uint32_t* epoch[kMaxPeers];      // per part 4 words: epochs completed (x2), CTA ticket counter (own entry only)
  uint32_t* err[kMaxPeers];        // barrier time-out word in device memory (only the own entry is used)
  uint32_t* err_host;              // its mapped pinned copy for the host
  unsigned long long timeout_ns;   // barrier time-out (DRL_B200_PEER_TIMEOUT_S)
};
struct PeerPlan {
  PeerTable t;
  OptState o;                      // the update's state (lr / step live here)
  int rank, world, nblk;
};
// one exchange instance over float4 range [beg4, end4) of the bucket; do_lr: also lr / global_step (last instance)
int peer_exchange(cudaStream_t s, const PeerPlan& pp, int part, int64_t beg4, int64_t end4, bool do_lr, int grid = 0);

}  // namespace drl
