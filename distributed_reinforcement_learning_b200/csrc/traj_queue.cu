// traj_queue.cu -- the device-resident queues behind drl_traj_queue_* (IMPALA trajectories), drl_r2d2_queue_* (R2D2
// sequences), drl_apex_queue_* (Ape-X local-buffer samples) and drl_a3c_queue_* (A3C unrolls) (include/drl_b200.h;
// layout and ordering in traj_queue.cuh).  Producers are policy-engine recorders (queue_recorder.cuh) and Ape-X actor
// buffers (apex_actor_buffer.cu), the consumers are drl_learner_stage_from_queue (learner.cu),
// drl_r2d2_replay_add_from_queue (r2d2_replay.cu), drl_apex_replay_add_from_queue (apex_replay.cu) and
// drl_a3c_stage_from_queue (apex.cu); no record byte crosses PCIe on its way into or out of a queue except what a
// recorder's commit uploads (reward and done; for A3C also the final next_state frames).
#include <string.h>

#include <algorithm>
#include <chrono>
#include <string>

#include "traj_queue.cuh"

using namespace drl;

namespace drl {

namespace {

size_t tq_align(size_t v) { return (v + 255) / 256 * 256; }

// every slot the n positions from reserved_total fall in is free for them (held slots and slots still holding an
// unpopped batch are not)
bool has_space(const QueueCore* q, int n) {
  long long p = q->reserved_total;
  const long long end = p + n;
  while (p < end) {
    const int slot = (int)((p / q->batch) % q->nslots), row0 = (int)(p % q->batch);
    const QueueCore::Slot& s = q->st[slot];
    if (s.held || s.reserved != row0) return false;
    p += q->batch - row0;
  }
  return true;
}

template <class Pred>
bool wait_for(std::condition_variable& cv, std::unique_lock<std::mutex>& lk, int timeout_ms, Pred pred) {
  if (timeout_ms < 0) {
    cv.wait(lk, pred);
    return true;
  }
  return cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
}

// the caller holds q->mu
int check_failed(const QueueCore* q) {
  if (!q->failed) return DRL_OK;
  set_error("%s is in the failed state: a commit failed after reserving its positions (%s)", q->name,
            q->failure.c_str());
  return DRL_ERR_STATE;
}

}  // namespace

int queue_core_init(QueueCore* q, int nfields, const size_t* sz, int capacity, int batch, int device) {
  q->nfields = nfields;
  q->batch = batch;
  q->device = device;
  q->nslots = (capacity + batch - 1) / batch + 1;
  size_t off = 0;
  for (int f = 0; f < nfields; ++f) {
    q->sz[f] = sz[f];
    q->off[f] = off;
    off = tq_align(off + (size_t)batch * sz[f]);
  }
  q->slot_bytes = off;
  q->st.resize(q->nslots);
  DRL_CUDA_CHECK(cudaSetDevice(device));
  DRL_CUDA_CHECK(cudaMalloc((void**)&q->base, q->slot_bytes * q->nslots));
  DRL_CUDA_CHECK(cudaMemset(q->base, 0, q->slot_bytes * q->nslots));
  // a slot takes at most `batch` commits (each writes at least one row) before it is popped
  for (auto& s : q->st) {
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&s.ev_release, cudaEventDisableTiming));
    s.ev_commit.assign(batch, nullptr);
    for (auto& e : s.ev_commit) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  DRL_CUDA_CHECK(cudaDeviceSynchronize());
  return DRL_OK;
}

void queue_core_release(QueueCore* q) {
  cudaSetDevice(q->device);
  for (auto& s : q->st) {
    if (s.ev_release) cudaEventSynchronize(s.ev_release);
    for (cudaEvent_t e : s.ev_commit) if (e) { cudaEventSynchronize(e); cudaEventDestroy(e); }
    if (s.ev_release) cudaEventDestroy(s.ev_release);
  }
  if (q->base) cudaFree(q->base);
  cudaGetLastError();
}

int queue_size(QueueCore* q) {
  std::lock_guard<std::mutex> lk(q->mu);
  return (int)(q->committed_total - q->popped_total);
}

int queue_read(QueueCore* q, int k, void* const* dst) {
  for (int f = 0; f < q->nfields; ++f)
    if (!dst[f]) { set_error("%s read: null output pointer", q->name); return DRL_ERR_INVALID; }
  std::lock_guard<std::mutex> lk(q->mu);
  DRL_TRY(check_failed(q));
  const long long size = q->committed_total - q->popped_total;
  if (k < 0 || k >= size) {
    set_error("%s read: k = %d is outside [0, %lld) (the queued %s)", q->name, k, size, q->items);
    return DRL_ERR_INVALID;
  }
  const long long p = q->popped_total + k;
  const int slot = (int)((p / q->batch) % q->nslots), row = (int)(p % q->batch);
  const QueueCore::Slot& s = q->st[slot];
  if (s.committed != s.reserved) {
    set_error("%s read: a commit into slot %d is still in progress", q->name, slot);
    return DRL_ERR_STATE;
  }
  DRL_CUDA_CHECK(cudaSetDevice(q->device));
  for (int i = 0; i < s.n_commit; ++i) DRL_CUDA_CHECK(cudaEventSynchronize(s.ev_commit[i]));
  for (int f = 0; f < q->nfields; ++f)
    DRL_CUDA_CHECK(cudaMemcpy(dst[f], q->field(slot, f) + (size_t)row * q->sz[f], q->sz[f], cudaMemcpyDeviceToHost));
  return DRL_OK;
}

void traj_queue_fail(QueueCore* q, const char* why) {
  {
    std::lock_guard<std::mutex> lk(q->mu);
    q->failed = true;
    q->failure = why;
  }
  q->cv_space.notify_all();
  q->cv_ready.notify_all();
}

int traj_queue_max_rows(const QueueCore* q) { return (q->nslots - 1) * q->batch + 1; }

int traj_queue_reserve(QueueCore* q, int n, int timeout_ms, std::vector<TrajSegment>* segs) {
  if (n < 1 || n > traj_queue_max_rows(q)) {
    set_error("%s: %d rows per commit can never fit (at most %d in this queue: %d slots of %d)", q->name, n,
              traj_queue_max_rows(q), q->nslots, q->batch);
    return DRL_ERR_INVALID;
  }
  std::unique_lock<std::mutex> lk(q->mu);
  if (!wait_for(q->cv_space, lk, timeout_ms, [&] { return q->failed || has_space(q, n); })) {
    set_error("%s commit: timed out (queue full)", q->name);
    return DRL_ERR_TIMEOUT;
  }
  DRL_TRY(check_failed(q));
  segs->clear();
  long long p = q->reserved_total;
  int src = 0;
  while (src < n) {
    const int slot = (int)((p / q->batch) % q->nslots), row0 = (int)(p % q->batch);
    const int rows = std::min(q->batch - row0, n - src);
    QueueCore::Slot& s = q->st[slot];
    segs->push_back(TrajSegment{slot, row0, rows, src, s.ev_commit[s.n_commit], s.ev_release});
    s.n_commit++;
    s.reserved += rows;
    p += rows;
    src += rows;
  }
  q->reserved_total = p;
  return DRL_OK;
}

void traj_queue_commit(QueueCore* q, const std::vector<TrajSegment>& segs) {
  std::lock_guard<std::mutex> lk(q->mu);
  bool ready = false;
  for (const TrajSegment& g : segs) {
    QueueCore::Slot& s = q->st[g.slot];
    s.committed += g.rows;
    q->committed_total += g.rows;
    ready = ready || s.committed == q->batch;
  }
  if (ready) q->cv_ready.notify_all();
}

int traj_queue_pop(QueueCore* q, int timeout_ms, int* slot, std::vector<cudaEvent_t>* ev_commit) {
  std::unique_lock<std::mutex> lk(q->mu);
  auto head = [&] { return (int)((q->popped_total / q->batch) % q->nslots); };
  auto ready = [&] {
    const QueueCore::Slot& s = q->st[head()];
    return !s.held && s.committed == q->batch;
  };
  if (!wait_for(q->cv_ready, lk, timeout_ms, [&] { return q->failed || ready(); })) {
    set_error("%s %s: timed out (fewer than batch %s queued)", q->name, q->pop_verb, q->items);
    return DRL_ERR_TIMEOUT;
  }
  DRL_TRY(check_failed(q));
  *slot = head();
  QueueCore::Slot& s = q->st[*slot];
  s.held = true;
  ev_commit->assign(s.ev_commit.begin(), s.ev_commit.begin() + s.n_commit);
  q->popped_total += q->batch;
  return DRL_OK;
}

int traj_queue_release(QueueCore* q, int slot, cudaStream_t s) {
  const cudaError_t e = cudaEventRecord(q->st[slot].ev_release, s);
  {
    std::lock_guard<std::mutex> lk(q->mu);
    QueueCore::Slot& st = q->st[slot];
    st.held = false;
    st.reserved = 0;
    st.committed = 0;
    st.n_commit = 0;
  }
  q->cv_space.notify_all();
  if (e != cudaSuccess) { set_error("%s release: %s", q->name, cudaGetErrorString(e)); return DRL_ERR_CUDA; }
  return DRL_OK;
}

}  // namespace drl

namespace {

// create's tail shared by both families: the core's slots, or the handle released with the error message kept
template <class Q>
int finish_create(Q* q, int nfields, const size_t* sz, int capacity, int batch, int device, Q** out,
                  int (*destroy)(Q*)) {
  const int rc = queue_core_init(q, nfields, sz, capacity, batch, device);
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    destroy(q);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = q;
  return DRL_OK;
}

int check_queue_device(int device) {
  if (drl_device_count() <= device || device < 0) {
    set_error("CUDA device %d not available (no CPU fallback)", device);
    return DRL_ERR_CUDA;
  }
  return DRL_OK;
}

// drl_apex_queue_create / drl_a3c_queue_create: one record of T transitions (or steps) in ApexIn order, one record per
// slot.  `family` prefixes the error messages ("apex queue", "a3c queue").
template <class Q>
int create_apex_layout_queue(const char* family, int trajectory, int num_action, int capacity, int device, Q** out,
                             int (*destroy)(Q*)) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (trajectory < 1 || trajectory > kApexQueueMaxT) {
    set_error("%s: trajectory must be in [1, %d] (got %d)", family, kApexQueueMaxT, trajectory);
    return DRL_ERR_INVALID;
  }
  if (num_action < 2 || num_action > 32) { set_error("%s: num_action must be in [2, 32] (got %d)", family, num_action); return DRL_ERR_INVALID; }
  if (capacity < 1) { set_error("%s: capacity must be >= 1 (got %d)", family, capacity); return DRL_ERR_INVALID; }
  DRL_TRY(check_queue_device(device));
  Q* q = new Q();
  q->name = family;
  q->pop_verb = "add_from_queue";
  q->items = "records";
  q->T = trajectory; q->A = num_action;
  const size_t T = trajectory;
  size_t sz[kApexQFields];
  sz[kApexQFrames] = 2 * T * Geo::FRAME;
  sz[kApexQPa2] = 2 * T * 4;
  sz[kApexQReward] = T * 4;
  sz[kApexQDone] = T;
  // one record per slot: a slot is an ApexIn of n = T rows
  return finish_create(q, kApexQFields, sz, capacity, 1, device, out, destroy);
}

// drl_apex_queue_read / drl_a3c_queue_read
int read_apex_layout_queue(QueueCore* q, int T, int k, uint8_t* state, uint8_t* next_state, int32_t* previous_action,
                           int32_t* action, float* reward, uint8_t* done) {
  if (!state || !next_state || !previous_action || !action) { set_error("%s read: null output pointer", q->name); return DRL_ERR_INVALID; }
  // the slot's frames and pa2 fields hold both halves; queue_read copies them into one block each, split below
  const size_t t = T;
  std::vector<uint8_t> frames(2 * t * Geo::FRAME);
  std::vector<int32_t> pa2(2 * t);
  void* const dst[kApexQFields] = {frames.data(), pa2.data(), reward, done};
  DRL_TRY(queue_read(q, k, dst));
  memcpy(state, frames.data(), t * Geo::FRAME);
  memcpy(next_state, frames.data() + t * Geo::FRAME, t * Geo::FRAME);
  memcpy(previous_action, pa2.data(), t * 4);
  memcpy(action, pa2.data() + t, t * 4);
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_traj_queue_create(int32_t trajectory, int32_t height, int32_t width, int32_t channels, int32_t num_action,
                          int32_t lstm_size, int32_t capacity, int32_t batch, int32_t device, drl_traj_queue** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (trajectory < 1 || height < 1 || width < 1 || channels < 1 || num_action < 1 || lstm_size < 1 || batch < 1 ||
      capacity < batch) {
    set_error("trajectory queue: invalid dimensions (capacity must be >= batch)");
    return DRL_ERR_INVALID;
  }
  DRL_TRY(check_queue_device(device));
  drl_traj_queue* q = new drl_traj_queue();
  q->name = "trajectory queue";
  q->pop_verb = "stage";
  q->items = "trajectories";
  q->T = trajectory; q->H = height; q->W = width; q->C = channels; q->A = num_action; q->L = lstm_size;
  const size_t T = trajectory;
  size_t sz[kTrajFields];
  sz[kTrajState] = T * height * width * channels;
  sz[kTrajReward] = T * 4;
  sz[kTrajDone] = T;
  sz[kTrajMu] = T * num_action * 4;
  sz[kTrajAction] = T * 4;
  sz[kTrajPa] = T * 4;
  sz[kTrajH] = T * lstm_size * 4;
  sz[kTrajC] = T * lstm_size * 4;
  return finish_create(q, kTrajFields, sz, capacity, batch, device, out, drl_traj_queue_destroy);
}

int drl_traj_queue_destroy(drl_traj_queue* q) {
  if (!q) return DRL_OK;
  queue_core_release(q);
  delete q;
  return DRL_OK;
}

int drl_traj_queue_size(drl_traj_queue* q) { return q ? queue_size(q) : 0; }

int drl_traj_queue_read(drl_traj_queue* q, int32_t k, uint8_t* state, float* reward, uint8_t* done,
                        float* behavior_policy, int32_t* action, int32_t* previous_action, float* previous_h,
                        float* previous_c) {
  if (!q) { set_error("null trajectory queue handle"); return DRL_ERR_INVALID; }
  void* const dst[kTrajFields] = {state, reward, done, behavior_policy, action, previous_action, previous_h, previous_c};
  return queue_read(q, k, dst);
}

int drl_r2d2_queue_create(int32_t seq_len, int32_t channels, int32_t num_action, int32_t capacity, int32_t batch,
                          int32_t device, drl_r2d2_queue** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (seq_len < 2) { set_error("r2d2 queue: seq_len must be >= 2 (got %d)", seq_len); return DRL_ERR_INVALID; }
  if (channels != 1 && channels != 4) { set_error("r2d2 queue: channels must be 1 or 4 (got %d)", channels); return DRL_ERR_INVALID; }
  if (num_action < 2 || num_action > 32) { set_error("r2d2 queue: num_action must be in [2, 32] (got %d)", num_action); return DRL_ERR_INVALID; }
  if (batch < 1 || capacity < batch) {
    set_error("r2d2 queue: invalid dimensions (batch must be >= 1 and capacity >= batch; got %d, %d)", batch, capacity);
    return DRL_ERR_INVALID;
  }
  DRL_TRY(check_queue_device(device));
  drl_r2d2_queue* q = new drl_r2d2_queue();
  q->name = "r2d2 queue";
  q->pop_verb = "add_from_queue";
  q->items = "sequences";
  q->S = seq_len; q->C = channels; q->A = num_action;
  q->frame = (size_t)Geo::IH * Geo::IW * channels;
  const size_t S = seq_len, L = 64;   // L: the R2D2 network's lstm_size (kR2L)
  size_t sz[kR2QFields];
  sz[kR2QFrames] = S * q->frame;
  sz[kR2QPa] = S * 4;
  sz[kR2QAction] = S * 4;
  sz[kR2QH] = L * 4;
  sz[kR2QC] = L * 4;
  sz[kR2QReward] = S * 4;
  sz[kR2QDone] = S;
  return finish_create(q, kR2QFields, sz, capacity, batch, device, out, drl_r2d2_queue_destroy);
}

int drl_r2d2_queue_destroy(drl_r2d2_queue* q) {
  if (!q) return DRL_OK;
  queue_core_release(q);
  delete q;
  return DRL_OK;
}

int drl_r2d2_queue_size(drl_r2d2_queue* q) { return q ? queue_size(q) : 0; }

int drl_r2d2_queue_read(drl_r2d2_queue* q, int32_t k, uint8_t* state, int32_t* previous_action, int32_t* action,
                        float* previous_h, float* previous_c, float* reward, uint8_t* done) {
  if (!q) { set_error("null r2d2 queue handle"); return DRL_ERR_INVALID; }
  void* const dst[kR2QFields] = {state, previous_action, action, previous_h, previous_c, reward, done};
  return queue_read(q, k, dst);
}

int drl_apex_queue_create(int32_t trajectory, int32_t num_action, int32_t capacity, int32_t device,
                          drl_apex_queue** out) {
  return create_apex_layout_queue("apex queue", trajectory, num_action, capacity, device, out, drl_apex_queue_destroy);
}

int drl_apex_queue_destroy(drl_apex_queue* q) {
  if (!q) return DRL_OK;
  queue_core_release(q);
  delete q;
  return DRL_OK;
}

int drl_apex_queue_size(drl_apex_queue* q) { return q ? queue_size(q) : 0; }

int drl_apex_queue_read(drl_apex_queue* q, int32_t k, uint8_t* state, uint8_t* next_state, int32_t* previous_action,
                        int32_t* action, float* reward, uint8_t* done) {
  if (!q) { set_error("null apex queue handle"); return DRL_ERR_INVALID; }
  return read_apex_layout_queue(q, q->T, k, state, next_state, previous_action, action, reward, done);
}

int drl_a3c_queue_create(int32_t trajectory, int32_t num_action, int32_t capacity, int32_t device,
                         drl_a3c_queue** out) {
  return create_apex_layout_queue("a3c queue", trajectory, num_action, capacity, device, out, drl_a3c_queue_destroy);
}

int drl_a3c_queue_destroy(drl_a3c_queue* q) {
  if (!q) return DRL_OK;
  queue_core_release(q);
  delete q;
  return DRL_OK;
}

int drl_a3c_queue_size(drl_a3c_queue* q) { return q ? queue_size(q) : 0; }

int drl_a3c_queue_read(drl_a3c_queue* q, int32_t k, uint8_t* state, uint8_t* next_state, int32_t* previous_action,
                       int32_t* action, float* reward, uint8_t* done) {
  if (!q) { set_error("null a3c queue handle"); return DRL_ERR_INVALID; }
  return read_apex_layout_queue(q, q->T, k, state, next_state, previous_action, action, reward, done);
}

}  // extern "C"
