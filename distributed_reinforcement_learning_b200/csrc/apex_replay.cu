// apex_replay.cu -- the Ape-X prioritized replay memory on the device, behind drl_apex_replay_* (include/drl_b200.h):
// buffer_queue.Memory (distributed_queue/buffer_queue.py:371-415) with its transitions in HBM, its sum tree on the
// device and the learner loop of train_apex.py:82-155 -- ingest with the learner's |td|, stratified sample, minibatch
// gather into a learner staging slot, step, priority update -- as kernels on the learner's compute stream, without a
// host round trip between steps (DESIGN.md section 10).  This file holds what depends on one record being a
// transition: the storage, the store and gather kernels and the ingest layout; the sum tree, the ordering of the
// memory's work and the sample / update / total / size / beta bodies are the shared core's (replay_core.cuh).
//
// The memory is independent of any one learner handle (apex.Agent may rebuild its learner for another batch size):
// every call that uses a learner takes it as an argument.
#include <string.h>

#include <mutex>
#include <string>

#include "apex_defs.cuh"
#include "replay_core.cuh"
#include "traj_queue.cuh"

using namespace drl;

namespace {

constexpr const char* kName = "apex replay";

// device ingest block of n transitions, packed like a learner's scratch slot for an n-row td_error:
// frames [2n] (s rows, then s' rows) | pa2 [2n] (previous_action, then action) | reward [n] | done [n] | weight [n] |
// error [n] (double, the caller's priorities when given)
struct IngestLayout {
  size_t fr, pa, rw, dn, wt, er, bytes;
  explicit IngestLayout(size_t n) {
    size_t off = 0;
    fr = off; off = align_up(off + 2 * n * Geo::FRAME, 256);
    pa = off; off = align_up(off + 2 * n * 4, 256);
    rw = off; off = align_up(off + n * 4, 256);
    dn = off; off = align_up(off + n, 256);
    wt = off; off = align_up(off + n * 4, 256);
    er = off; off = align_up(off + n * 8, 256);
    bytes = off;
  }
};

}  // namespace

// the sum tree, the ordering and the sample / update state are the shared core's (replay_core.cuh)
struct drl_apex_replay : ReplayCore {
  // the transitions, zero-initialised: a leaf past n_entries reached through float drift gathers a defined record
  uint8_t* state = nullptr;            // [capacity][84,84,4]
  uint8_t* next_state = nullptr;       // [capacity][84,84,4]
  int32_t *previous_action = nullptr, *action = nullptr;
  float* reward = nullptr;
  uint8_t* done = nullptr;
};

namespace {

int check_replay(const drl_apex_replay* r) { return replay_check(r, kName); }

// a learner argument: an Ape-X (not A3C) handle on the memory's device
int check_learner(const drl_apex_replay* r, const drl_apex* h) {
  DRL_TRY(check_handle(h, "apex"));
  if (h->algo != 0) { set_error("apex replay: the learner is an A3C handle, the memory serves Ape-X learners"); return DRL_ERR_INVALID; }
  if (h->device != r->device) {
    set_error("apex replay: the learner is on device %d, the memory on device %d", h->device, r->device);
    return DRL_ERR_INVALID;
  }
  return DRL_OK;
}

}  // namespace

namespace drl {

// Copies n ingested transitions (device block `in`, packed with s' rows at row n) into the storage rows
// (first + i) mod capacity.  Grid (n, 2): block (i, 0) copies state row i and the scalars, block (i, 1) next_state.
__global__ void __launch_bounds__(256) apex_replay_store_kernel(const ApexIn in, int n, int64_t first, int64_t capacity,
                                                                 uint8_t* __restrict__ state,
                                                                 uint8_t* __restrict__ next_state,
                                                                 int32_t* __restrict__ previous_action,
                                                                 int32_t* __restrict__ action,
                                                                 float* __restrict__ reward,
                                                                 uint8_t* __restrict__ done) {
  kernel_prologue();
  const int i = blockIdx.x, half = blockIdx.y;
  const int64_t row = (first + i) % capacity;
  const uint4* src = reinterpret_cast<const uint4*>(in.frames + ((size_t)half * n + i) * Geo::FRAME);
  uint4* dst = reinterpret_cast<uint4*>((half ? next_state : state) + (size_t)row * Geo::FRAME);
  for (int k = threadIdx.x; k < Geo::FRAME / 16; k += blockDim.x) dst[k] = src[k];
  if (half == 0 && threadIdx.x == 0) {
    previous_action[row] = in.pa2[i];
    action[row] = in.pa2[n + i];
    reward[row] = in.reward[i];
    done[row] = in.done[i];
  }
}

// The minibatch of a training step: the sampled rows data_index[0, B) of the storage into a learner slot in the
// layout drl_apex_stage writes (state rows, then next_state rows; previous_action, then action; reward; done).  The
// importance weights are written by the sample kernel.  Grid (B, 2) like the store kernel.
__global__ void __launch_bounds__(256) apex_replay_gather_kernel(const int64_t* __restrict__ data_index, int B,
                                                                  const uint8_t* __restrict__ state,
                                                                  const uint8_t* __restrict__ next_state,
                                                                  const int32_t* __restrict__ previous_action,
                                                                  const int32_t* __restrict__ action,
                                                                  const float* __restrict__ reward,
                                                                  const uint8_t* __restrict__ done, ApexIn out) {
  kernel_prologue();
  const int i = blockIdx.x, half = blockIdx.y;
  const int64_t row = data_index[i];
  const uint4* src = reinterpret_cast<const uint4*>((half ? next_state : state) + (size_t)row * Geo::FRAME);
  uint4* dst = reinterpret_cast<uint4*>(out.frames + ((size_t)half * B + i) * Geo::FRAME);
  for (int k = threadIdx.x; k < Geo::FRAME / 16; k += blockDim.x) dst[k] = src[k];
  if (half == 0 && threadIdx.x == 0) {
    out.pa2[i] = previous_action[row];
    out.pa2[B + i] = action[row];
    out.reward[i] = reward[row];
    out.done[i] = done[row];
  }
}

}  // namespace drl

extern "C" {

int drl_apex_replay_create(int32_t device, int64_t capacity, drl_apex_replay** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  DRL_TRY(replay_check_create(kName, device, capacity));
  drl_apex_replay* r = new drl_apex_replay();
  r->family = kName;
  int rc = [&]() -> int {
    const size_t C = (size_t)capacity;
    DRL_TRY(replay_core_init(r, device, capacity));
    DRL_TRY(dev_alloc(r, &r->state, C * Geo::FRAME));
    DRL_TRY(dev_alloc(r, &r->next_state, C * Geo::FRAME));
    DRL_TRY(dev_alloc(r, &r->previous_action, C));
    DRL_TRY(dev_alloc(r, &r->action, C));
    DRL_TRY(dev_alloc(r, &r->reward, C));
    DRL_TRY(dev_alloc(r, &r->done, C));
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_apex_replay_destroy(r);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = r;
  return DRL_OK;
}

int drl_apex_replay_destroy(drl_apex_replay* r) {
  if (!r) return DRL_OK;
  replay_core_release(r);
  delete r;
  return DRL_OK;
}

int drl_apex_replay_add(drl_apex_replay* r, drl_apex* learner, int32_t n, const uint8_t* state,
                        const uint8_t* next_state, const int32_t* previous_action, const int32_t* action,
                        const float* reward, const uint8_t* done, const double* error) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!state || !next_state || !previous_action || !action || !reward || !done) { set_error("apex replay add: null input pointer"); return DRL_ERR_INVALID; }
  if (n < 1 || n > r->capacity) { set_error("apex replay add: n must be in [1, capacity = %lld]", (long long)r->capacity); return DRL_ERR_INVALID; }
  if (!error && !learner) { set_error("apex replay add: without errors the learner computes them (null learner)"); return DRL_ERR_INVALID; }
  std::unique_lock<std::recursive_mutex> llk;
  if (learner) {
    DRL_TRY(check_learner(r, learner));
    llk = std::unique_lock<std::recursive_mutex>(learner->mu);
    if (n > learner->B) { set_error("apex replay add: n = %d exceeds the learner's batch %d", n, learner->B); return DRL_ERR_INVALID; }
  }
  if (learner)       // the learner's embedding gathers these rows
    for (int i = 0; i < n; ++i)
      if (previous_action[i] < 0 || previous_action[i] >= learner->A || action[i] < 0 || action[i] >= learner->A) {
        set_error("apex replay add: an action of transition %d is not in [0, %d)", i, learner->A);
        return DRL_ERR_INVALID;
      }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  const IngestLayout L(n);
  DRL_TRY(replay_ensure_ingest(r, L.bytes));
  uint8_t* h = r->ingest.h;
  memcpy(h + L.fr, state, (size_t)n * Geo::FRAME);
  memcpy(h + L.fr + (size_t)n * Geo::FRAME, next_state, (size_t)n * Geo::FRAME);
  memcpy(h + L.pa, previous_action, (size_t)n * 4);
  memcpy(h + L.pa + (size_t)n * 4, action, (size_t)n * 4);
  memcpy(h + L.rw, reward, (size_t)n * 4);
  memcpy(h + L.dn, done, (size_t)n);
  float* w = reinterpret_cast<float*>(h + L.wt);
  for (int i = 0; i < n; ++i) w[i] = 1.0f;
  if (error) memcpy(h + L.er, error, (size_t)n * 8);
  uint8_t* d = r->d_ingest;
  const ApexIn in{d + L.fr, reinterpret_cast<int32_t*>(d + L.pa), reinterpret_cast<float*>(d + L.rw), d + L.dn,
                  reinterpret_cast<float*>(d + L.wt)};
  const cudaStream_t s = learner ? learner->compute : r->stream;
  DRL_TRY(replay_begin(r, s));
  DRL_CUDA_CHECK(cudaMemcpyAsync(d, h, L.bytes, cudaMemcpyHostToDevice, s));
  DRL_CUDA_CHECK(cudaEventRecord(r->ingest.ev, s));
  if (!error) {
    // agent/apex.py:116-133 on the device: the learner's forward + TD path, |td| stays in td_dev
    DRL_TRY(enqueue_forward_td(learner, in, n, false, nullptr, nullptr));
    learner->last_n = n;
  }
  prof_mark(s, "replay_store");
  DRL_CUDA_CHECK((launch_k(apex_replay_store_kernel, dim3(n, 2), 256, 0, s, in, n, r->cursor, r->capacity, r->state,
                           r->next_state, r->previous_action, r->action, r->reward, r->done)));
  DRL_TRY(replay_launch_update(r, s, n, nullptr, r->cursor, error ? reinterpret_cast<const double*>(d + L.er) : nullptr,
                               error ? nullptr : learner->td_dev));
  DRL_TRY(replay_end(r, s));
  replay_advance(r, n);
  return DRL_OK;
}

int drl_apex_replay_add_from_queue(drl_apex_replay* r, drl_apex* learner, drl_apex_queue* q, int32_t timeout_ms) {
  DRL_TRY(check_replay(r));
  if (!q) { set_error("null apex queue handle"); return DRL_ERR_INVALID; }
  {
    std::lock_guard<std::recursive_mutex> lk(r->mu);
    DRL_TRY(check_learner(r, learner));
    std::lock_guard<std::recursive_mutex> llk(learner->mu);
    if (q->device != r->device) {
      set_error("apex replay add_from_queue: the queue is on device %d, the memory on device %d", q->device, r->device);
      return DRL_ERR_INVALID;
    }
    if (q->A != learner->A) {
      set_error("apex replay add_from_queue: the queue has num_action %d, the learner %d", q->A, learner->A);
      return DRL_ERR_INVALID;
    }
    // drl_apex_replay_add chunks a longer record; the slot is read in place and cannot be
    if (q->T > learner->B) {
      set_error("apex replay add_from_queue: the queue's trajectory %d exceeds the learner's batch %d", q->T, learner->B);
      return DRL_ERR_INVALID;
    }
    if (q->T > r->capacity) {
      set_error("apex replay add_from_queue: the queue's trajectory %d exceeds the memory's capacity %lld", q->T,
                (long long)r->capacity);
      return DRL_ERR_INVALID;
    }
  }
  // wait for a record without either lock: actor threads sync their engines from this learner meanwhile
  int qs = 0;
  std::vector<cudaEvent_t> ev_commit;
  DRL_TRY(traj_queue_pop(q, timeout_ms, &qs, &ev_commit));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  std::lock_guard<std::recursive_mutex> llk(learner->mu);
  NvtxRange nv("drl:apex_replay_add_from_queue");
  const int n = q->T;
  const cudaStream_t s = learner->compute;
  // The slot is an ApexIn of n = T rows as it is: the learner and the store read it in place.  Its weight is null, which
  // the TD kernel reads as 1, the value drl_apex_replay_add stages.  Nothing here checks the actions on the host: the
  // queue's only producers are actor buffers, whose appends check every previous action and action.
  const ApexIn in{q->field(qs, kApexQFrames), reinterpret_cast<int32_t*>(q->field(qs, kApexQPa2)),
                  reinterpret_cast<float*>(q->field(qs, kApexQReward)), q->field(qs, kApexQDone), nullptr};
  const int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(r->device));
    DRL_TRY(replay_begin(r, s));
    for (cudaEvent_t e : ev_commit) DRL_CUDA_CHECK(cudaStreamWaitEvent(s, e, 0));
    DRL_TRY(enqueue_forward_td(learner, in, n, false, nullptr, nullptr));
    learner->last_n = n;
    prof_mark(s, "replay_store");
    DRL_CUDA_CHECK((launch_k(apex_replay_store_kernel, dim3(n, 2), 256, 0, s, in, n, r->cursor, r->capacity, r->state,
                             r->next_state, r->previous_action, r->action, r->reward, r->done)));
    return replay_launch_update(r, s, n, nullptr, r->cursor, nullptr, learner->td_dev);
  }();
  // the queue slot goes back to the producers either way (their gathers into it wait for its release event)
  const int rc_release = traj_queue_release(q, qs, s);
  DRL_TRY(rc);
  DRL_TRY(rc_release);
  DRL_TRY(replay_end(r, s));
  replay_advance(r, n);
  return DRL_OK;
}

int drl_apex_replay_step_async(drl_apex_replay* r, drl_apex* learner, int32_t slot, const double* u01) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  DRL_TRY(check_learner(r, learner));
  std::lock_guard<std::recursive_mutex> llk(learner->mu);
  DRL_TRY(check_slot(learner, slot));
  const int B = learner->B;
  const ApexIn& in = learner->in[slot];
  // Memory.sample -> gather -> step -> Memory.update with the step's |td| (train_apex.py:118-154)
  return replay_step(r, learner, slot, u01, in.weight, learner->td_dev, [&](cudaStream_t s) -> int {
    prof_mark(s, "replay_gather");
    DRL_CUDA_CHECK((launch_k(apex_replay_gather_kernel, dim3(B, 2), 256, 0, s, r->d_data_index, B, r->state,
                             r->next_state, r->previous_action, r->action, r->reward, r->done, in)));
    return DRL_OK;
  });
}

int drl_apex_replay_sample(drl_apex_replay* r, int32_t n, const double* u01, int64_t* tree_index, int64_t* data_index,
                           double* priority, double* is_weight) {
  return replay_sample(r, kName, n, u01, tree_index, data_index, priority, is_weight);
}

int drl_apex_replay_update(drl_apex_replay* r, int32_t n, const int64_t* tree_index, const double* error) {
  return replay_update(r, kName, n, tree_index, error);
}

int drl_apex_replay_last_sample(drl_apex_replay* r, int64_t* tree_index, double* priority, double* is_weight) {
  return replay_last_sample(r, kName, tree_index, priority, is_weight);
}

int drl_apex_replay_read(drl_apex_replay* r, int64_t data_index, int32_t n, uint8_t* state, uint8_t* next_state,
                         int32_t* previous_action, int32_t* action, float* reward, uint8_t* done) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || data_index < 0 || data_index + n > r->capacity) {
    set_error("apex replay read: rows [%lld, %lld) are not inside [0, %lld)", (long long)data_index,
              (long long)(data_index + n), (long long)r->capacity);
    return DRL_ERR_INVALID;
  }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  const size_t i = (size_t)data_index, m = (size_t)n;
  auto cp = [](void* dst, const void* src, size_t bytes) { return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost); };
  if (state) DRL_CUDA_CHECK(cp(state, r->state + i * Geo::FRAME, m * Geo::FRAME));
  if (next_state) DRL_CUDA_CHECK(cp(next_state, r->next_state + i * Geo::FRAME, m * Geo::FRAME));
  if (previous_action) DRL_CUDA_CHECK(cp(previous_action, r->previous_action + i, m * 4));
  if (action) DRL_CUDA_CHECK(cp(action, r->action + i, m * 4));
  if (reward) DRL_CUDA_CHECK(cp(reward, r->reward + i, m * 4));
  if (done) DRL_CUDA_CHECK(cp(done, r->done + i, m));
  return DRL_OK;
}

int drl_apex_replay_total(drl_apex_replay* r, double* total) { return replay_total(r, kName, total); }
int drl_apex_replay_size(drl_apex_replay* r, int64_t* n_entries) { return replay_size(r, kName, n_entries); }
int drl_apex_replay_beta(drl_apex_replay* r, double* beta) { return replay_beta(r, kName, beta); }

}  // extern "C"
