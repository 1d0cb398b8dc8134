// policy_core.cu -- the network-independent half of the batched policy engines (policy_core.cuh) and of their queue
// recorders (queue_recorder.cuh).
#include <string.h>

#include <algorithm>
#include <string>

#include "policy_core.cuh"
#include "queue_recorder.cuh"

namespace drl {
namespace {

using Lock = std::lock_guard<std::recursive_mutex>;

// "drl:<family>_<call>" with the family's spaces as underscores (drl:r2d2_policy_set_params)
std::string range_name(const char* family, const char* call) {
  std::string s = std::string("drl:") + family + "_" + call;
  std::replace(s.begin(), s.end(), ' ', '_');
  return s;
}

// the action-embedding table and the conv weight images of the current parameters, on the engine's stream
int refresh_derived(PolicyCore* h) {
  const TrunkLayout& pl = *h->layout;
  const float* P = h->params;
  DRL_TRY(emb_forward(h->stream, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, h->e1, h->table, h->A));
  return h->conv_images(h->stream, pl, P, h->img_conv2, h->img_conv3);
}

}  // namespace

int policy_check_device(int device) {
  if (drl_device_count() <= device || device < 0) {
    set_error("CUDA device %d not available (no CPU fallback)", device);
    return DRL_ERR_CUDA;
  }
  return DRL_OK;
}

int policy_core_init(PolicyCore* h, int (*set_attributes)(), size_t zpart_floats, size_t in_bytes, size_t out_bytes) {
  const size_t MB = h->max_batch;
  const int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(h->device));
    DRL_TRY(set_attributes());
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_ready, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_copied, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreate(&h->ev_start));
    DRL_CUDA_CHECK(cudaEventCreate(&h->ev_stop));
    DRL_TRY(dev_alloc(h, &h->params, (size_t)h->layout->padded_total));
    size_t wb[WeightImages::kCount];
    weight_image_sizes(wb);
    DRL_TRY(dev_alloc(h, &h->img_conv2, wb[1]));
    DRL_TRY(dev_alloc(h, &h->img_conv3, wb[2]));
    DRL_TRY(dev_alloc(h, &h->e1, (size_t)h->A * Geo::EMB));
    DRL_TRY(dev_alloc(h, &h->table, (size_t)h->A * Geo::EMB));
    DRL_TRY(dev_alloc(h, &h->a1, MB * 400 * 32));
    DRL_TRY(dev_alloc(h, &h->a2, MB * 81 * 64));
    DRL_TRY(dev_alloc(h, &h->a3, MB * Geo::FLAT));
    DRL_TRY(dev_alloc(h, &h->a1p, 2 * MB * 400 * 32));
    DRL_TRY(dev_alloc(h, &h->a2p, 2 * MB * 81 * 64));
    DRL_TRY(dev_alloc(h, &h->zpart, zpart_floats));
    DRL_TRY(dev_alloc(h, &h->d_in, in_bytes));
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_in, in_bytes, cudaHostAllocDefault));
    memset(h->h_in, 0, in_bytes);
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_out, out_bytes, cudaHostAllocMapped));
    memset(h->h_out, 0, out_bytes);
    DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_out, h->h_out, 0));
    h->graphs.assign(MB + 1, nullptr);
    DRL_TRY(refresh_derived(h));   // zero parameters until set_params / sync
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    policy_core_release(h);
    set_error("%s", keep.c_str());
  }
  return rc;
}

void policy_core_release(PolicyCore* h) {
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto g : h->graphs) if (g) cudaGraphExecDestroy(g);
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_in) cudaFreeHost(h->h_in);
  if (h->h_out) cudaFreeHost(h->h_out);
  for (cudaEvent_t e : {h->ev_ready, h->ev_copied, h->ev_start, h->ev_stop}) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  cudaGetLastError();
}

int policy_run_act(PolicyCore* h, int n) {
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->stream));
  if (h->use_cuda_graph) {
    if (!h->graphs[n]) {
      DRL_TRY(h->enqueue_act(h, n));
      DRL_TRY(capture_graph(h->stream, [&] { return h->enqueue_act(h, n); }, &h->graphs[n]));
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graphs[n], h->stream));
  } else {
    DRL_TRY(h->enqueue_act(h, n));
  }
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->stream));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->timed = true;
  h->last_n = n;
  return DRL_OK;
}

int policy_check_n(const PolicyCore* h, int n, bool inputs_given) {
  if (n < 1 || n > h->max_batch) { set_error("act: n must be in [1, %d] (got %d)", h->max_batch, n); return DRL_ERR_INVALID; }
  if (!inputs_given) { set_error("act: null input pointer"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int policy_check_actions(const PolicyCore* h, int n, const int32_t* previous_action, const int32_t* explore) {
  for (int i = 0; i < n; ++i) {
    if (previous_action && (previous_action[i] < 0 || previous_action[i] >= h->A)) {
      set_error("act: previous_action[%d] = %d is outside [0, %d)", i, previous_action[i], h->A);
      return DRL_ERR_INVALID;
    }
    if (explore && (explore[i] < -1 || explore[i] >= h->A)) {
      set_error("act: explore_action[%d] = %d is outside [-1, %d)", i, explore[i], h->A);
      return DRL_ERR_INVALID;
    }
  }
  return DRL_OK;
}

void policy_stage_explore(uint8_t* dst, const int32_t* explore, int n) {
  if (explore) memcpy(dst, explore, (size_t)n * 4);
  else memset(dst, 0xff, (size_t)n * 4);   // -1: greedy
}

int policy_check(const PolicyCore* h, const char* family) {
  if (!h) { set_error("null %s handle", family); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int policy_param_count(const PolicyCore* h, const char* family, int64_t* n) {
  DRL_TRY(policy_check(h, family));
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->layout->packed_total;
  return DRL_OK;
}

int policy_set_params(PolicyCore* h, const char* family, const float* host_flat, int64_t n) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  const FlatLayout& pl = *h->layout;
  if (!host_flat || n != pl.packed_total) {
    set_error("set_params: expected %lld floats, got %lld", (long long)pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv(range_name(family, "set_params").c_str());
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  std::vector<float> flat((size_t)pl.padded_total);
  DRL_TRY(upload_flat(h->stream, flat.data(), pl, h->params, host_flat, 0.0f));
  DRL_TRY(refresh_derived(h));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  return DRL_OK;
}

int policy_get_params(PolicyCore* h, const char* family, float* host_flat, int64_t n) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  const FlatLayout& pl = *h->layout;
  if (!host_flat || n != pl.packed_total) {
    set_error("get_params: expected %lld floats, got %lld", (long long)pl.packed_total, (long long)n);
    return DRL_ERR_INVALID;
  }
  NvtxRange nv(range_name(family, "get_params").c_str());
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  std::vector<float> flat((size_t)pl.padded_total);
  return download_flat(h->stream, flat.data(), pl, h->params, host_flat);
}

int policy_sync(PolicyCore* h, const char* family, const void* learner, const std::function<int()>& snapshot) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  if (!learner) { set_error("null learner handle"); return DRL_ERR_INVALID; }
  NvtxRange nv(range_name(family, "sync").c_str());
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_TRY(snapshot());
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  return refresh_derived(h);
}

int policy_last_act_ms(PolicyCore* h, const char* family, float* ms) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (!h->timed) { set_error("last_act_ms: no act call has run yet"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

int policy_read_buffer(PolicyCore* h, const char* family, const char* name, float* host_dst, int64_t n) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  if (!name || !host_dst) { set_error("null argument"); return DRL_ERR_INVALID; }
  if (h->last_n < 1) { set_error("read_buffer: no act call has run yet"); return DRL_ERR_STATE; }
  const size_t m = h->last_n, A = h->A;
  const struct { const char* name; const float* p; size_t count; } tab[] = {
      {"a1", h->a1, m * 400 * 32}, {"a2", h->a2, m * 81 * 64}, {"a3", h->a3, m * Geo::FLAT},
      {"e1", h->e1, A * Geo::EMB}, {"table", h->table, A * Geo::EMB},
      {"zpart", h->zpart, (size_t)h->splits * m * h->zpart_cols}};
  for (const auto& e : tab) {
    if (strcmp(e.name, name) != 0) continue;
    if ((size_t)n != e.count) { set_error("read_buffer(%s): expected %zu floats, got %lld", name, e.count, (long long)n); return DRL_ERR_INVALID; }
    DRL_CUDA_CHECK(cudaSetDevice(h->device));
    DRL_CUDA_CHECK(cudaMemcpyAsync(host_dst, e.p, e.count * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
    return DRL_OK;
  }
  set_error("read_buffer: unknown buffer '%s'", name);
  return DRL_ERR_INVALID;
}

int policy_buffer_dims(PolicyCore* h, const char* family, int32_t* out) {
  DRL_TRY(policy_check(h, family));
  Lock lk(h->mu);
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  out[0] = h->last_n;
  out[1] = h->splits;
  out[2] = h->zpart_cols;
  return DRL_OK;
}

// ---- recorders ---------------------------------------------------------------------------------------------------
int recorder_core_init(RecorderCore* r) {
  DRL_CUDA_CHECK(cudaSetDevice(r->engine->device));
  size_t off = 0;
  for (int f = 0; f < r->q->nfields; ++f) {
    r->off[f] = off;
    off = align_up(off + (size_t)r->n * r->q->sz[f], 256);
  }
  DRL_TRY(dev_alloc(r, &r->staging, off));
  DRL_TRY(dev_alloc(r, &r->d_t, 1));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&r->h_t, sizeof(int32_t), cudaHostAllocDefault));
  *r->h_t = 0;
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&r->h_rd, (size_t)r->n * r->T * 5, cudaHostAllocDefault));
  return DRL_OK;
}

void recorder_core_release(RecorderCore* r) {
  if (r->engine && r->engine->stream) cudaStreamSynchronize(r->engine->stream);
  if (r->graph) cudaGraphExecDestroy(r->graph);
  for (void* p : r->allocs) cudaFree(p);
  if (r->h_t) cudaFreeHost(r->h_t);
  if (r->h_rd) cudaFreeHost(r->h_rd);
  cudaGetLastError();
}

int recorder_check_step(const RecorderCore* r) {
  if (r->t >= r->T) {
    set_error("recorder act: all %d steps of the unroll are recorded (commit them first)", r->T);
    return DRL_ERR_STATE;
  }
  return DRL_OK;
}

int recorder_run_act(RecorderCore* r, const std::function<int()>& enqueue_step) {
  PolicyCore* h = r->engine;
  *r->h_t = r->t;
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->stream));
  if (h->use_cuda_graph) {
    if (!r->graph) {
      DRL_TRY(enqueue_step());   // eager pass first: attributes and tensor maps outside capture (idempotent)
      DRL_TRY(capture_graph(h->stream, enqueue_step, &r->graph));
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(r->graph, h->stream));
  } else {
    DRL_TRY(enqueue_step());
  }
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->stream));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->stream));
  h->timed = true;
  h->last_n = r->n;
  r->t++;
  return DRL_OK;
}

int recorder_commit(RecorderCore* r, const float* reward, const uint8_t* done, int timeout_ms,
                    const std::function<int()>& before_copies) {
  if (!reward || !done) { set_error("recorder commit: null argument"); return DRL_ERR_INVALID; }
  PolicyCore* h = r->engine;
  {
    Lock lk(h->mu);
    if (r->t != r->T) {
      set_error("recorder commit: %d of %d steps recorded (commit follows step %s)", r->t, r->T, r->last_step);
      return DRL_ERR_STATE;
    }
  }
  // reserve without the engine's lock: a learner thread may sync this engine while the commit waits for space
  std::vector<TrajSegment> segs;
  DRL_TRY(traj_queue_reserve(r->q, r->n, timeout_ms, &segs));
  Lock lk(h->mu);
  NvtxRange nv(r->commit_range);
  QueueCore* q = r->q;
  cudaStream_t s = h->stream;
  const size_t nT = (size_t)r->n * r->T;
  const int rc = [&]() -> int {
    // h_rd is free: every act since the previous commit waited for the stream
    memcpy(r->h_rd, reward, nT * 4);
    memcpy(r->h_rd + nT * 4, done, nT);
    DRL_CUDA_CHECK(cudaSetDevice(h->device));
    DRL_CUDA_CHECK(cudaMemcpyAsync(r->field(r->f_reward), r->h_rd, nT * 4, cudaMemcpyHostToDevice, s));
    DRL_CUDA_CHECK(cudaMemcpyAsync(r->field(r->f_done), r->h_rd + nT * 4, nT, cudaMemcpyHostToDevice, s));
    if (before_copies) DRL_TRY(before_copies());
    for (const TrajSegment& g : segs) {
      DRL_CUDA_CHECK(cudaStreamWaitEvent(s, g.ev_release, 0));
      for (int f = 0; f < q->nfields; ++f)
        DRL_CUDA_CHECK(cudaMemcpyAsync(q->field(g.slot, f) + (size_t)g.row0 * q->sz[f],
                                       r->field(f) + (size_t)g.src0 * q->sz[f], (size_t)g.rows * q->sz[f],
                                       cudaMemcpyDeviceToDevice, s));
      DRL_CUDA_CHECK(cudaEventRecord(g.ev_commit, s));
    }
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    // the reserved positions will never be filled: rather than leave every producer and the consumer waiting behind
    // them, the queue goes into its failed state (every later reserve / pop / read returns DRL_ERR_STATE)
    traj_queue_fail(q, get_error());
    return rc;
  }
  traj_queue_commit(q, segs);
  r->t = 0;
  return DRL_OK;
}

int recorder_reset(RecorderCore* r) {
  Lock lk(r->engine->mu);
  r->t = 0;
  return DRL_OK;
}

}  // namespace drl
