// learner.cu -- the IMPALA learner handle behind the C-ABI (include/drl_b200.h), on the learner-handle core
// (learner_core.cuh): RMSProp slots, activations, V-trace, the staging views and the NVLink peer exchange.
// Replaces impala.Agent's learner graph and Agent.train (agent/impala.py:11-103,132-148).
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "learner_core.cuh"
#include "traj_queue.cuh"

// NVTX ranges (NvtxRange, kernels.h) around the host-side phases of a step: stage (H2D enqueue), forward,
// vtrace_losses, backward, exchange, update.  Inside a CUDA-graph replay the phases are one cudaGraphLaunch, so the
// ranges mark the capture / eager enqueue and the replay as a whole ("step(graph)").

using namespace drl;

struct drl_learner : LearnerCore {
  drl_learner_config cfg{};
  int T = 0, A = 0, M = 0, Mb = 0;
  ParamLayout pl{};
  std::vector<Inputs> in;    // the staging slots' fields, caller's batch-major layout
  cudaStream_t xchg = nullptr;
  cudaEvent_t ev_lstm_grads = nullptr, ev_xchg_done = nullptr;   // early part of the peer exchange (stream xchg)
  int peer_early_ctas = 64;   // grid of the early exchange instance (DRL_B200_PEER_EARLY_CTAS; 0 = no early part)
  cudaStream_t side2 = nullptr;   // second side lane (small head weight gradients)
  cudaEvent_t fj2[4] = {};
  float* ms = nullptr;
  Acts act{};
  Bwd bwd{};
  WeightImages wimg{};
  VtraceOut vt{};
  OptState opt{};
  Recurrence rec{};          // recurrent mode (cfg.recurrent = 1): cluster counts of the recurrence kernels
  // gradient exchange over NVLink peer memory (peer.cu); off until drl_learner_peer_import
  bool peer_on = false;
  int peer_nblk = 132 * 4;
  uint8_t* comm = nullptr;                   // [reduced | partials | flags | epochs | err], own cudaMalloc (IPC-exported)
  size_t comm_bytes = 0, off_partials = 0, off_flags = 0, off_epoch = 0, off_err = 0;
  PeerPlan plan{};                           // peer table + the update's OptState on the reduced buffer
  std::vector<void*> peer_opened;            // bases returned by cudaIpcOpenMemHandle
  uint32_t* h_peer_err = nullptr;            // pinned copy of the barrier time-out word
  bool failed = false;                       // a peer barrier timed out: the replica is out of step with its peers and
                                             // refuses every further step / state read (drl_learner_wait reported it)
};

namespace {

constexpr const char* kName = "learner";

int check_not_failed(const drl_learner* h) {
  if (h->failed) {
    set_error("learner handle is in the failed state (a peer-exchange barrier timed out): parameters and optimizer "
              "state are not readable and no further step can run");
    return DRL_ERR_STATE;
  }
  return DRL_OK;
}

Streams streams_of(const drl_learner* h) {
  Streams st = h->streams();
  st.side2 = h->side2;
  for (int i = 0; i < 4; ++i) st.ev2[i] = h->fj2[i];
  st.ev_lstm_grads = (h->peer_on && h->peer_early_ctas > 0) ? h->ev_lstm_grads : nullptr;
  return st;
}

// retile = true: (re)build the weight images first.  A training step always does (the parameters changed in the
// previous apply); the forward-only entry points only when the images are stale.
int enqueue_forward(drl_learner* h, const Inputs& in, int B, int T, bool retile) {
  return net_forward(streams_of(h), h->pl, h->params, h->wimg, in, h->act, B, T, h->mode, retile, h->rec);
}

int fwd_bwd(LearnerCore* core, int slot, int* launches) {
  drl_learner* h = static_cast<drl_learner*>(core);
  const Inputs& in = h->in[slot];
  {
    NvtxRange r("drl:forward");
    DRL_TRY(enqueue_forward(h, in, h->B, h->T, true));
  }
  VtraceCfg vc{h->cfg.discount_factor, h->cfg.baseline_loss_coef, h->cfg.entropy_coef, h->cfg.reward_clipping};
  prof_mark(h->compute, "vtrace_losses");
  {
    NvtxRange r("drl:vtrace_losses");
    DRL_TRY(vtrace_losses(h->compute, vc, h->act.policy, h->act.value, in, h->vt, h->bwd.dlogits, h->bwd.dv, h->B,
                          h->T, h->A));
  }
  NvtxRange r("drl:backward");
  DRL_TRY(net_backward(streams_of(h), h->pl, h->params, h->wimg, h->grads, in, h->act, h->bwd, h->B, h->T, h->mode,
                       h->rec));
  if (launches) *launches += forward_launch_count() + 1 + backward_launch_count();   // + the V-trace/loss kernel
  return DRL_OK;
}

// RMSProp on the local bucket, or with the peer exchange on, on the reduced one.  No grad_scale: the IMPALA losses are
// batch sums, so the summed bucket of the replicas is the gradient of the global batch.
// local_only: the single-replica update on the local bucket even when the peer exchange is on (profiling on one rank)
// early: the backward pass of THIS enqueue recorded ev_lstm_grads (one-graph step): part 0 of the exchange overlaps it
int update(LearnerCore* core, int out_row, float /*grad_scale*/, bool local_only, bool early) {
  drl_learner* h = static_cast<drl_learner*>(core);
  early = early && h->peer_on && h->par && h->peer_early_ctas > 0;
  OptState o_local = h->opt, o_peer = h->plan.o;
  o_local.out = o_peer.out = h->d_out + 8 * out_row;
  if (h->peer_on && !local_only) {
    prof_mark(h->compute, "peer_exchange");
    {
      NvtxRange r("drl:exchange");
      // part 0: [lstm_w .. end) incl. the loss sums -- 96 % of the bucket.  In the one-graph step it runs on its own stream
      // behind the LSTM weight gradient (ev_lstm_grads), i.e. under the rest of the backward pass, with a small grid so that
      // the convolution kernels never queue behind it; otherwise right here.  part 1: [0 .. lstm_w), after the backward pass.
      const int64_t split4 = h->pl.lstm_w / 4, end4 = h->pl.padded_total / 4 + 1;
      if (early) {
        DRL_CUDA_CHECK(cudaStreamWaitEvent(h->xchg, h->ev_lstm_grads, 0));
        DRL_TRY(peer_exchange(h->xchg, h->plan, 0, split4, end4, false, h->peer_early_ctas));
        DRL_CUDA_CHECK(cudaEventRecord(h->ev_xchg_done, h->xchg));
        DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, h->ev_xchg_done, 0));
      } else {
        DRL_TRY(peer_exchange(h->compute, h->plan, 0, split4, end4, false, h->peer_early_ctas));
      }
      DRL_TRY(peer_exchange(h->compute, h->plan, 1, 0, split4, true, 132));
    }
    prof_mark(h->compute, "optimizer(rmsprop)");
    NvtxRange r("drl:update");
    DRL_TRY(optimizer_update_only(h->compute, o_peer));
    prof_mark(h->compute, "end");
  } else {
    prof_mark(h->compute, "optimizer(norm+rmsprop)");
    NvtxRange r("drl:update");
    DRL_TRY(optimizer_apply(h->compute, o_local));
    prof_mark(h->compute, "end");
  }
  // no D2H copy node: the update kernel stores the 8 scalars straight into mapped pinned memory (h_out); a memcpy
  // at the end of the graph sat in the ~20 us gap between two steps (tools/timeline.py --back-to-back)
  return DRL_OK;
}

// the scalars of result row r; a peer barrier time-out puts the handle into the failed state
int step_out(drl_learner* h, const float* r, drl_step_out* out) {
  if (h->peer_on && h->h_peer_err && *h->h_peer_err) {
    h->failed = true;
    set_error("peer exchange: rank %d never reached the barrier within %.0f s (DRL_B200_PEER_TIMEOUT_S); this replica "
              "skipped the update and is out of step with its peers: destroy the handle",
              (int)*h->h_peer_err - 1, (double)h->plan.t.timeout_ns * 1e-9);
    return DRL_ERR_STATE;
  }
  if (out) {
    out->pi_loss = r[0];
    out->baseline_loss = r[1];
    out->entropy = r[2];
    out->learning_rate = r[3];
    out->grad_norm = r[4];
    out->total_loss = r[5];
    out->step = step_of(r);
  }
  return DRL_OK;
}

}  // namespace

int drl::impala_params_snapshot(drl_learner* h, int device, int num_action, cudaStream_t dst_stream, float* dst,
                                cudaEvent_t ev_ready, cudaEvent_t ev_copied) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  if (h->A != num_action) {
    set_error("sync: the learner has num_action %d, the policy %d", h->A, num_action);
    return DRL_ERR_INVALID;
  }
  return learner_params_snapshot(h, kName, device, dst_stream, dst, ev_ready, ev_copied);
}

extern "C" {

int drl_learner_create(const drl_learner_config* cfg, drl_learner** out) {
  if (!cfg || !out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (cfg->height != Geo::IH || cfg->width != Geo::IW || cfg->channels != Geo::IC) {
    set_error("only the reference input geometry 84x84x4 is supported (got %dx%dx%d)", cfg->height, cfg->width,
              cfg->channels);
    return DRL_ERR_INVALID;
  }
  if (cfg->lstm_size != Geo::L) { set_error("only lstm_size 256 is supported (got %d)", cfg->lstm_size); return DRL_ERR_INVALID; }
  if (cfg->trajectory < 3 || cfg->trajectory > 32) { set_error("trajectory must be in [3,32]"); return DRL_ERR_INVALID; }
  if (cfg->num_action < 2 || cfg->num_action > 32) { set_error("num_action must be in [2,32]"); return DRL_ERR_INVALID; }
  if (cfg->batch < 1) { set_error("batch must be >= 1"); return DRL_ERR_INVALID; }
  if (cfg->reward_clipping != DRL_REWARD_ABS_ONE && cfg->reward_clipping != DRL_REWARD_SOFT_ASYMMETRIC) {
    set_error("reward_clipping must be DRL_REWARD_ABS_ONE or DRL_REWARD_SOFT_ASYMMETRIC");   // utils.py:45
    return DRL_ERR_INVALID;
  }
  if (cfg->math_mode < 0 || cfg->math_mode > 5 || cfg->math_mode == 4) {
    set_error("math_mode must be 0 (default), 1 (FP32 FFMA), 2 (wgmma 3xTF32), 3 (same, persistent kernels) "
              "or 5 (wgmma with 16-bit split operands)");
    return DRL_ERR_INVALID;
  }
  if (cfg->recurrent != 0 && cfg->recurrent != 1) {
    set_error("recurrent must be 0 (one LSTM step from each step's recorded state) or 1 (unroll through the trajectory)");
    return DRL_ERR_INVALID;
  }
  if (cfg->recurrent && (cfg->math_mode == 1 || cfg->math_mode == 3)) {
    set_error("recurrent = 1 runs in math mode 5 (default) or 2; math mode %d is not supported with it", cfg->math_mode);
    return DRL_ERR_INVALID;
  }
  if (drl_device_count() <= cfg->device) { set_error("CUDA device %d not available (no CPU fallback)", cfg->device); return DRL_ERR_CUDA; }

  drl_learner* h = new drl_learner();
  h->cfg = *cfg;
  h->device = cfg->device;
  h->num_slots = cfg->num_slots < 1 ? 2 : cfg->num_slots;
  h->use_cuda_graph = cfg->use_cuda_graph != 0;
  h->mode = (cfg->math_mode == 0) ? DRL_DEFAULT_MATH_MODE_IMPALA : cfg->math_mode;
  h->B = cfg->batch; h->T = cfg->trajectory; h->A = cfg->num_action;
  h->M = h->B * h->T; h->Mb = h->B * (h->T - 2);
  h->pl.init(h->A);
  h->layout = &h->pl;
  h->fwd_bwd = fwd_bwd;
  h->update = update;
  int rc = [&]() -> int {
    const size_t M = h->M, Mb = h->Mb, A = h->A, NP = h->pl.padded_total, BT = (size_t)h->B * h->T;
    size_t off = 0;
    const size_t o_frames = off; off = align_up(off + BT * Geo::FRAME, 256);
    const size_t o_rew = off; off = align_up(off + BT * 4, 256);
    const size_t o_act = off; off = align_up(off + BT * 4, 256);
    const size_t o_done = off; off = align_up(off + BT, 256);
    const size_t o_mu = off; off = align_up(off + BT * A * 4, 256);
    const size_t o_pa = off; off = align_up(off + BT * 4, 256);
    const size_t o_h = off; off = align_up(off + BT * Geo::L * 4, 256);
    const size_t o_c = off; off = align_up(off + BT * Geo::L * 4, 256);
    DRL_TRY(learner_core_init(h, off));
    for (const LearnerSlot& s : h->slots)
      h->in.push_back(Inputs{s.base + o_frames, reinterpret_cast<float*>(s.base + o_rew),
                             reinterpret_cast<int32_t*>(s.base + o_act), s.base + o_done,
                             reinterpret_cast<float*>(s.base + o_mu), reinterpret_cast<int32_t*>(s.base + o_pa),
                             reinterpret_cast<float*>(s.base + o_h), reinterpret_cast<float*>(s.base + o_c)});
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->xchg, cudaStreamNonBlocking));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_lstm_grads, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_xchg_done, cudaEventDisableTiming));
    if (const char* e = getenv("DRL_B200_PEER_EARLY_CTAS")) h->peer_early_ctas = atoi(e);
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side2, cudaStreamNonBlocking));
    for (int i = 0; i < 4; ++i) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->fj2[i], cudaEventDisableTiming));
    DRL_TRY(dev_alloc(h, &h->ms, NP));
    {  // RMSProp slots start at ONE (TF1 RMSPropOptimizer._create_slots)
      std::vector<float> ones(NP, 1.0f);
      DRL_CUDA_CHECK(cudaMemcpy(h->ms, ones.data(), NP * sizeof(float), cudaMemcpyHostToDevice));
    }
    Acts& a = h->act;
    DRL_TRY(alloc_trunk_acts(h, a, M, A, h->mode == 5));
    DRL_TRY(dev_alloc(h, &a.zpart, (size_t)kLstmSplits * M * Geo::G4));
    DRL_TRY(dev_alloc(h, &a.gates, M * Geo::G4));
    DRL_TRY(dev_alloc(h, &a.c1, M * Geo::L));
    DRL_TRY(dev_alloc(h, &a.tc1, M * Geo::L));
    DRL_TRY(dev_alloc(h, &a.h1, M * Geo::L));
    DRL_TRY(dev_alloc(h, &a.hid1, 2 * M * Geo::HID));
    DRL_TRY(dev_alloc(h, &a.hid2, 2 * M * Geo::HID));
    DRL_TRY(dev_alloc(h, &a.logits, M * A));
    DRL_TRY(dev_alloc(h, &a.policy, M * A));
    DRL_TRY(dev_alloc(h, &a.value, M));
    if (cfg->recurrent) {
      DRL_TRY(impala_recurrence_setup(&h->rec));
      DRL_TRY(dev_alloc(h, &a.zx, M * Geo::G4));
      DRL_TRY(dev_alloc(h, &a.hin, M * Geo::L));
      DRL_TRY(dev_alloc(h, &a.cin, M * Geo::L));
    }
    if (h->mode == 5) {
      DRL_TRY(dev_alloc(h, &a.img_xt, lstm_image_bytes(1, (int)M, (int)Mb)));
      DRL_TRY(dev_alloc(h, &h->bwd.img_dzt, lstm_image_bytes(3, (int)M, (int)Mb)));
    }
    Bwd& b = h->bwd;
    DRL_TRY(dev_alloc(h, &b.dlogits, Mb * 32));
    DRL_TRY(dev_alloc(h, &b.dv, Mb * 32));
    DRL_TRY(dev_alloc(h, &b.dhid2, 2 * Mb * Geo::HID));
    DRL_TRY(dev_alloc(h, &b.dhid1, 2 * Mb * Geo::HID));
    DRL_TRY(dev_alloc(h, &b.dh_part, 2 * Mb * Geo::L));
    DRL_TRY(dev_alloc(h, &b.dz, Mb * Geo::G4));
    DRL_TRY(alloc_trunk_bwd(h, b, Mb, A, Geo::IC, h->mode != 5, h->mode == 5));
    b.wg_part_floats = trunk_partial_floats((int)Mb, Geo::IC);
    DRL_TRY(dev_alloc(h, &b.emb_scratch, (size_t)16 * 32 * 256));
    {
      size_t wb[WeightImages::kCount];
      weight_image_sizes(wb);
      for (int i = 0; i < WeightImages::kCount; ++i) DRL_TRY(dev_alloc(h, &h->wimg.img[i], wb[i]));
    }
    VtraceOut& v = h->vt;
    const size_t nt = (size_t)h->B * (h->T - 2);
    DRL_TRY(dev_alloc(h, &v.vs, nt));
    DRL_TRY(dev_alloc(h, &v.clipped_rho, nt));
    DRL_TRY(dev_alloc(h, &v.vs_plus_1, nt));
    DRL_TRY(dev_alloc(h, &v.pg_adv, nt));
    DRL_TRY(dev_alloc(h, &v.loss_partials, (size_t)cdiv(h->B, 4) * 3));
    DRL_TRY(dev_alloc(h, &v.ticket, 1));
    v.loss_sums = h->loss;
    OptState& o = h->opt;
    o.params = h->params; o.ms = h->ms; o.grads = h->grads; o.n = (int64_t)NP;
    o.nblk = 132 * 4;
    o.npart = o.nblk;
    o.wait_flags = nullptr; o.wait_epoch = nullptr; o.wait_world = 0; o.wait_err = nullptr; o.wait_parts = 0;
    o.wait_err_host = nullptr; o.wait_timeout_ns = 0;
    DRL_TRY(dev_alloc(h, &o.norm_partials, o.nblk));
    o.step = h->d_step; o.lr_cur = h->d_lr; o.out = h->d_out; o.loss_sums = v.loss_sums;
    o.start_lr = cfg->start_learning_rate; o.end_lr = cfg->end_learning_rate; o.learning_frame = cfg->learning_frame;
    o.clip_norm = cfg->gradient_clip_norm; o.baseline_coef = cfg->baseline_loss_coef; o.entropy_coef = cfg->entropy_coef;
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_learner_destroy(h);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = h;
  return DRL_OK;
}

int drl_learner_destroy(drl_learner* h) {
  if (!h) return DRL_OK;
  learner_core_release(h);
  for (void* p : h->peer_opened) cudaIpcCloseMemHandle(p);
  if (h->comm) cudaFree(h->comm);
  if (h->h_peer_err) cudaFreeHost(h->h_peer_err);
  for (int i = 0; i < 4; ++i) if (h->fj2[i]) cudaEventDestroy(h->fj2[i]);
  if (h->side2) cudaStreamDestroy(h->side2);
  if (h->xchg) cudaStreamDestroy(h->xchg);
  if (h->ev_lstm_grads) cudaEventDestroy(h->ev_lstm_grads);
  if (h->ev_xchg_done) cudaEventDestroy(h->ev_xchg_done);
  cudaGetLastError();
  delete h;
  return DRL_OK;
}

int drl_learner_param_count(const drl_learner* h, int64_t* n) { return learner_param_count(h, kName, n); }
int drl_learner_set_params(drl_learner* h, const float* host_flat, int64_t n) {
  return learner_set_params(h, kName, host_flat, n);
}
int drl_learner_get_params(drl_learner* h, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  return learner_get_params(h, kName, host_flat, n);
}
int drl_learner_set_opt_state(drl_learner* h, const float* host_ms_flat, int64_t n, int64_t step) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!host_ms_flat || n != h->pl.packed_total) { set_error("set_opt_state: expected %lld floats", (long long)h->pl.packed_total); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(learner_upload(h, h->ms, host_ms_flat, 1.0f));
  long long st = step;
  DRL_CUDA_CHECK(cudaMemcpy(h->d_step, &st, sizeof(st), cudaMemcpyHostToDevice));
  return DRL_OK;
}
int drl_learner_get_opt_state(drl_learner* h, float* host_ms_flat, int64_t n, int64_t* step) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  if (n != h->pl.packed_total) { set_error("get_opt_state: expected %lld floats", (long long)h->pl.packed_total); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  if (host_ms_flat) DRL_TRY(learner_download(h, h->ms, host_ms_flat));
  if (step) {
    long long st = 0;
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
    DRL_CUDA_CHECK(cudaMemcpy(&st, h->d_step, sizeof(st), cudaMemcpyDeviceToHost));
    *step = st;
  }
  return DRL_OK;
}
int drl_learner_get_grads(drl_learner* h, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  return learner_get_grads(h, kName, h->peer_on ? reinterpret_cast<float*>(h->comm) : h->grads, host_flat, n);
}

int drl_learner_stage(drl_learner* h, int32_t slot, const uint8_t* state, const float* reward, const int32_t* action,
                      const uint8_t* done, const float* behavior_policy, const int32_t* previous_action,
                      const float* initial_h, const float* initial_c) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  if (!state || !reward || !action || !done || !behavior_policy || !previous_action || !initial_h || !initial_c) {
    set_error("stage: null input pointer");
    return DRL_ERR_INVALID;
  }
  DRL_TRY(set_device(h));
  NvtxRange nvtx_r("drl:stage");
  LearnerSlot& s = h->slots[slot];
  const Inputs& in = h->in[slot];
  const size_t BT = (size_t)h->B * h->T;
  // do not overwrite a slot the compute stream is still reading
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, s.consumed, 0));
  auto cp = [&](const void* dst, const void* src, size_t bytes) -> cudaError_t {
    return cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, h->copy);
  };
  DRL_CUDA_CHECK(cp(in.frames, state, BT * Geo::FRAME));
  DRL_CUDA_CHECK(cp(in.reward, reward, BT * 4));
  DRL_CUDA_CHECK(cp(in.action, action, BT * 4));
  DRL_CUDA_CHECK(cp(in.done, done, BT));
  DRL_CUDA_CHECK(cp(in.mu, behavior_policy, BT * h->A * 4));
  DRL_CUDA_CHECK(cp(in.pa, previous_action, BT * 4));
  DRL_CUDA_CHECK(cp(in.h0, initial_h, BT * Geo::L * 4));
  DRL_CUDA_CHECK(cp(in.c0, initial_c, BT * Geo::L * 4));
  DRL_CUDA_CHECK(cudaEventRecord(s.staged, h->copy));
  s.has_data = true;
  return DRL_OK;
}

int drl_learner_stage_from_queue(drl_learner* h, int32_t slot, drl_traj_queue* q, int32_t timeout_ms) {
  DRL_TRY(check_handle(h, kName));
  if (!q) { set_error("null trajectory queue handle"); return DRL_ERR_INVALID; }
  {
    std::lock_guard<std::recursive_mutex> lk(h->mu);
    DRL_TRY(check_slot(h, slot));
    if (q->device != h->device) {
      set_error("stage_from_queue: the queue is on device %d, the learner on device %d", q->device, h->device);
      return DRL_ERR_INVALID;
    }
    if (q->batch != h->B || q->T != h->T || q->A != h->A) {
      set_error("stage_from_queue: the queue has batch %d, trajectory %d, num_action %d; the learner %d, %d, %d",
                q->batch, q->T, q->A, h->B, h->T, h->A);
      return DRL_ERR_INVALID;
    }
    if (q->H != Geo::IH || q->W != Geo::IW || q->C != Geo::IC || q->L != Geo::L) {
      set_error("stage_from_queue: the queue stores %dx%dx%d frames and lstm %d, the learner takes %dx%dx%d and %d",
                q->H, q->W, q->C, q->L, Geo::IH, Geo::IW, Geo::IC, Geo::L);
      return DRL_ERR_INVALID;
    }
  }
  // wait for a full batch without the learner's lock: actor threads sync their engines from this learner meanwhile
  int qs = 0;
  std::vector<cudaEvent_t> ev_commit;
  DRL_TRY(traj_queue_pop(q, timeout_ms, &qs, &ev_commit));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  NvtxRange nvtx_r("drl:stage_from_queue");
  LearnerSlot& s = h->slots[slot];
  const Inputs& in = h->in[slot];
  const int rc = [&]() -> int {
    DRL_TRY(set_device(h));
    // do not overwrite a slot the compute stream is still reading; do not read rows whose commit copies are pending
    DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, s.consumed, 0));
    for (cudaEvent_t e : ev_commit) DRL_CUDA_CHECK(cudaStreamWaitEvent(h->copy, e, 0));
    const void* dst[kTrajFields] = {in.frames, in.reward, in.done, in.mu, in.action, in.pa, in.h0, in.c0};
    for (int f = 0; f < kTrajFields; ++f)
      DRL_CUDA_CHECK(cudaMemcpyAsync(const_cast<void*>(dst[f]), q->field(qs, f), (size_t)q->batch * q->sz[f],
                                     cudaMemcpyDeviceToDevice, h->copy));
    DRL_CUDA_CHECK(cudaEventRecord(s.staged, h->copy));
    s.has_data = true;
    return DRL_OK;
  }();
  // the queue slot goes back to the producers either way (their copies into it wait for its release event)
  const int rc_release = traj_queue_release(q, qs, h->copy);
  return rc != DRL_OK ? rc : rc_release;
}

int drl_learner_forward_backward(drl_learner* h, int32_t slot) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  return learner_forward_backward(h, kName, slot);
}

int drl_learner_grad_bucket(drl_learner* h, void** dev_ptr, int64_t* count) {
  return learner_grad_bucket(h, kName, dev_ptr, count);
}

int drl_learner_reduced_bucket(drl_learner* h, void** dev_ptr, int64_t* count) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (dev_ptr) *dev_ptr = h->peer_on ? static_cast<void*>(h->comm) : static_cast<void*>(h->grads);
  if (count) *count = h->pl.padded_total + 4;
  return DRL_OK;
}

int drl_learner_apply(drl_learner* h) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  return learner_apply(h, kName, 1.0f);
}

// ---- gradient exchange over NVLink peer memory (peer.cu) -------------------------------------------------------
int drl_learner_peer_export(drl_learner* h, void* handles, int64_t bytes) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!handles || bytes != 2 * (int64_t)sizeof(cudaIpcMemHandle_t)) { set_error("peer_export: expected a %d-byte buffer", (int)(2 * sizeof(cudaIpcMemHandle_t))); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  if (!h->comm) {
    const size_t red = align_up((size_t)(h->pl.padded_total + 4) * sizeof(float), 256);
    h->off_partials = red;
    h->off_flags = h->off_partials + align_up((size_t)kPeerParts * kMaxPeers * h->peer_nblk * sizeof(float), 256);
    h->off_epoch = h->off_flags + 2 * kPeerParts * kMaxPeers * sizeof(uint32_t);
    h->off_err = h->off_epoch + 4 * kPeerParts * sizeof(uint32_t);
    h->comm_bytes = h->off_err + 256;
    DRL_CUDA_CHECK(cudaMalloc((void**)&h->comm, h->comm_bytes));
    DRL_CUDA_CHECK(cudaMemset(h->comm, 0, h->comm_bytes));
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_peer_err, sizeof(uint32_t), cudaHostAllocMapped));   // zero-copy too
    *h->h_peer_err = 0;
  }
  cudaIpcMemHandle_t hd[2];
  DRL_CUDA_CHECK(cudaIpcGetMemHandle(&hd[0], h->grads));
  DRL_CUDA_CHECK(cudaIpcGetMemHandle(&hd[1], h->comm));
  memcpy(handles, hd, sizeof(hd));
  return DRL_OK;
}

int drl_learner_peer_import(drl_learner* h, int32_t rank, int32_t world, const void* all_handles, int64_t bytes) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (world < 2 || world > kMaxPeers || rank < 0 || rank >= world) { set_error("peer_import: bad rank %d / world %d (max %d)", rank, world, kMaxPeers); return DRL_ERR_INVALID; }
  if (!all_handles || bytes != (int64_t)world * 2 * (int64_t)sizeof(cudaIpcMemHandle_t)) { set_error("peer_import: expected world x %d bytes", (int)(2 * sizeof(cudaIpcMemHandle_t))); return DRL_ERR_INVALID; }
  if (!h->comm) { set_error("peer_import before peer_export"); return DRL_ERR_STATE; }
  if (h->peer_on) { set_error("peer exchange already set up"); return DRL_ERR_STATE; }
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  const cudaIpcMemHandle_t* hd = static_cast<const cudaIpcMemHandle_t*>(all_handles);
  for (int p = 0; p < world; ++p) {
    float* bucket = h->grads;
    uint8_t* comm = h->comm;
    if (p != rank) {
      void *b = nullptr, *c = nullptr;
      DRL_CUDA_CHECK(cudaIpcOpenMemHandle(&b, hd[2 * p], cudaIpcMemLazyEnablePeerAccess));
      h->peer_opened.push_back(b);
      DRL_CUDA_CHECK(cudaIpcOpenMemHandle(&c, hd[2 * p + 1], cudaIpcMemLazyEnablePeerAccess));
      h->peer_opened.push_back(c);
      bucket = static_cast<float*>(b);
      comm = static_cast<uint8_t*>(c);
    }
    h->plan.t.bucket[p] = bucket;
    h->plan.t.reduced[p] = reinterpret_cast<float*>(comm);
    h->plan.t.partials[p] = reinterpret_cast<float*>(comm + h->off_partials);
    h->plan.t.flags[p] = reinterpret_cast<uint32_t*>(comm + h->off_flags);
    h->plan.t.epoch[p] = reinterpret_cast<uint32_t*>(comm + h->off_epoch);
    h->plan.t.err[p] = reinterpret_cast<uint32_t*>(comm + h->off_err);
  }
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->plan.t.err_host, h->h_peer_err, 0));   // host-visible copy
  {
    const char* e = getenv("DRL_B200_PEER_TIMEOUT_S");
    double sec = e ? atof(e) : 600.0;
    if (!(sec > 0.0)) sec = 600.0;
    h->plan.t.timeout_ns = (unsigned long long)(sec * 1e9);
  }
  h->plan.rank = rank;
  h->plan.world = world;
  h->plan.nblk = h->peer_nblk;
  OptState& po = h->plan.o;
  po = h->opt;
  po.grads = reinterpret_cast<float*>(h->comm);
  po.norm_partials = reinterpret_cast<float*>(h->comm + h->off_partials);
  po.npart = kPeerParts * world * h->peer_nblk;
  po.loss_sums = reinterpret_cast<float*>(h->comm) + h->pl.padded_total;
  po.wait_flags = h->plan.t.flags[rank];
  po.wait_epoch = h->plan.t.epoch[rank];
  po.wait_world = world;
  po.wait_err = h->plan.t.err[rank];
  po.wait_err_host = h->plan.t.err_host;
  po.wait_timeout_ns = h->plan.t.timeout_ns;
  po.wait_parts = kPeerParts;
  // graphs captured so far do not contain the exchange
  for (auto& g : h->graph_step) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  if (h->graph_apply) { cudaGraphExecDestroy(h->graph_apply); h->graph_apply = nullptr; }
  h->peer_on = true;
  return DRL_OK;
}

int drl_learner_peer_disable(drl_learner* h) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  for (void* p : h->peer_opened) cudaIpcCloseMemHandle(p);
  h->peer_opened.clear();
  cudaGetLastError();
  if (h->peer_on) {
    for (auto& g : h->graph_step) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
    if (h->graph_apply) { cudaGraphExecDestroy(h->graph_apply); h->graph_apply = nullptr; }
  }
  h->peer_on = false;
  return DRL_OK;
}

int drl_learner_stream(drl_learner* h, void** stream) { return learner_stream(h, kName, stream); }

int drl_learner_step_async(drl_learner* h, int32_t slot) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_not_failed(h));
  return learner_step_async(h, kName, slot);
}

int drl_learner_wait(drl_learner* h, drl_step_out* out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);     // the scalar row stays valid while it is read
  const float* r = nullptr;
  DRL_TRY(learner_wait(h, kName, &r));
  return step_out(h, r, out);
}

int drl_learner_wait_slot(drl_learner* h, int32_t slot, drl_step_out* out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const float* r = nullptr;
  DRL_TRY(learner_wait_slot(h, kName, slot, &r));
  return step_out(h, r, out);
}

int drl_learner_step(drl_learner* h, int32_t slot, drl_step_out* out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(drl_learner_step_async(h, slot));
  return drl_learner_wait(h, out);
}

int drl_learner_forward(drl_learner* h, int32_t slot, float* policy, float* value) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  LearnerSlot& s = h->slots[slot];
  if (!s.has_data) { set_error("slot %d has not been staged", slot); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, s.staged, 0));
  DRL_TRY(enqueue_forward(h, h->in[slot], h->B, h->T, h->images_stale));
  h->images_stale = false;
  DRL_CUDA_CHECK(cudaEventRecord(s.consumed, h->compute));
  // time-major device rows -> batch-major host arrays
  const int B = h->B, T = h->T, A = h->A;
  std::vector<float> pol((size_t)B * T * A), val((size_t)B * T);
  DRL_CUDA_CHECK(cudaMemcpyAsync(pol.data(), h->act.policy, pol.size() * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaMemcpyAsync(val.data(), h->act.value, val.size() * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  for (int t = 0; t < T; ++t)
    for (int b = 0; b < B; ++b) {
      const size_t m = (size_t)t * B + b, s2 = (size_t)b * T + t;
      if (policy) memcpy(policy + s2 * A, pol.data() + m * A, A * sizeof(float));
      if (value) value[s2] = val[m];
    }
  return DRL_OK;
}

int drl_learner_taps(drl_learner* h, float* vs, float* clipped_rho, float* vs_plus_1, float* pg_advantage) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(set_device(h));
  const size_t n = (size_t)h->B * (h->T - 2) * sizeof(float);
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  if (vs) DRL_CUDA_CHECK(cudaMemcpy(vs, h->vt.vs, n, cudaMemcpyDeviceToHost));
  if (clipped_rho) DRL_CUDA_CHECK(cudaMemcpy(clipped_rho, h->vt.clipped_rho, n, cudaMemcpyDeviceToHost));
  if (vs_plus_1) DRL_CUDA_CHECK(cudaMemcpy(vs_plus_1, h->vt.vs_plus_1, n, cudaMemcpyDeviceToHost));
  if (pg_advantage) DRL_CUDA_CHECK(cudaMemcpy(pg_advantage, h->vt.pg_adv, n, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_learner_read_buffer(drl_learner* h, const char* name, float* host_dst, int64_t n) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!name || !host_dst) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  const size_t M = h->M, Mb = h->Mb, A = h->A;
  const NamedBuffer tab[] = {
      {"a1", h->act.a1, M * 400 * 32}, {"a2", h->act.a2, M * 81 * 64}, {"a3", h->act.a3, M * Geo::FLAT},
      {"emb", h->act.table, A * Geo::EMB}, {"e1", h->act.e1, A * Geo::EMB},
      {"gates", h->act.gates, M * Geo::G4}, {"h1", h->act.h1, M * Geo::L}, {"c1", h->act.c1, M * Geo::L},
      {"hid1", h->act.hid1, 2 * M * Geo::HID}, {"hid2", h->act.hid2, 2 * M * Geo::HID},
      {"logits", h->act.logits, M * A}, {"policy", h->act.policy, M * A}, {"value", h->act.value, M},
      {"dlogits", h->bwd.dlogits, Mb * 32}, {"dv", h->bwd.dv, Mb * 32}, {"dhid2", h->bwd.dhid2, 2 * Mb * Geo::HID},
      {"dhid1", h->bwd.dhid1, 2 * Mb * Geo::HID}, {"dh_part", h->bwd.dh_part, 2 * Mb * Geo::L},
      {"dz", h->bwd.dz, Mb * Geo::G4}, {"hin", h->act.hin, M * Geo::L}, {"cin", h->act.cin, M * Geo::L},
      {"hout", h->rec.on() ? h->act.h1 : nullptr, M * Geo::L}, {"tc", h->rec.on() ? h->act.tc1 : nullptr, M * Geo::L},
      {"da3", h->bwd.da3, Mb * Geo::FLAT}, {"du", h->bwd.du, Mb * Geo::EMB},
      {"da2", h->bwd.da2, Mb * 81 * 64}, {"da1", h->bwd.da1, Mb * 400 * 32},
      // math mode 5's 16-bit planes, [hi | lo] bf16 (2 x 2 bytes per element: the buffer's count in 4-byte words)
      {"a1_plane", reinterpret_cast<float*>(h->act.a1p), M * 400 * 32},
      {"a2_plane", reinterpret_cast<float*>(h->act.a2p), M * 81 * 64},
      {"da3_plane", reinterpret_cast<float*>(h->bwd.da3p), Mb * Geo::FLAT},
      {"da2_plane", reinterpret_cast<float*>(h->bwd.da2p), Mb * 81 * 64}};
  return read_named_buffer(h, tab, sizeof(tab) / sizeof(tab[0]), name, host_dst, n);
}

int drl_learner_act(drl_learner* h, int32_t n, const uint8_t* state, const int32_t* previous_action,
                    const float* h_in, const float* c_in, float* policy, float* h_out, float* c_out) {
  DRL_TRY(check_handle(h, kName));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (n < 1 || n > h->M) { set_error("act: n must be in [1, %d]", h->M); return DRL_ERR_INVALID; }
  if (!state || !previous_action || !h_in || !c_in) { set_error("act: null input pointer"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  // reuse staging slot 0 as an [n, 1] batch (B = n, T = 1 makes the time-major/batch-major remap the identity); one
  // LSTM step from the given state in either mode
  const Inputs& in = h->in[0];
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->copy));
  auto cp = [&](const void* dst, const void* src, size_t bytes) -> cudaError_t {
    return cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, h->compute);
  };
  DRL_CUDA_CHECK(cp(in.frames, state, (size_t)n * Geo::FRAME));
  DRL_CUDA_CHECK(cp(in.pa, previous_action, (size_t)n * 4));
  DRL_CUDA_CHECK(cp(in.h0, h_in, (size_t)n * Geo::L * 4));
  DRL_CUDA_CHECK(cp(in.c0, c_in, (size_t)n * Geo::L * 4));
  h->slots[0].has_data = false;   // the slot no longer holds a training batch
  DRL_TRY(net_forward(streams_of(h), h->pl, h->params, h->wimg, in, h->act, n, 1, h->mode, h->images_stale,
                      Recurrence{}));
  h->images_stale = false;
  if (policy) DRL_CUDA_CHECK(cudaMemcpyAsync(policy, h->act.policy, (size_t)n * h->A * 4, cudaMemcpyDeviceToHost, h->compute));
  if (h_out) DRL_CUDA_CHECK(cudaMemcpyAsync(h_out, h->act.h1, (size_t)n * Geo::L * 4, cudaMemcpyDeviceToHost, h->compute));
  if (c_out) DRL_CUDA_CHECK(cudaMemcpyAsync(c_out, h->act.c1, (size_t)n * Geo::L * 4, cudaMemcpyDeviceToHost, h->compute));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  return DRL_OK;
}

int drl_learner_profile_step(drl_learner* h, int32_t slot, char* names, int64_t names_len, float* ms,
                             int32_t max_kernels, int32_t* count) {
  return learner_profile_step(h, kName, slot, names, names_len, ms, max_kernels, count);
}
int drl_learner_last_step_ms(drl_learner* h, float* ms) { return learner_last_step_ms(h, kName, ms); }
int drl_learner_launches_per_step(const drl_learner* h, int32_t* n) { return learner_launches_per_step(h, kName, n); }

}  // extern "C"
