// apex_replay.cu -- the Ape-X prioritized replay memory on the device, behind drl_apex_replay_* (include/drl_b200.h):
// buffer_queue.Memory (distributed_queue/buffer_queue.py:371-415) with its transitions in HBM, its sum tree on the
// device (replay_tree.cuh) and the learner loop of train_apex.py:82-155 -- ingest with the learner's |td|, stratified
// sample, minibatch gather into a learner staging slot, step, priority update -- as kernels on the learner's compute
// stream, without a host round trip between steps (DESIGN.md section 10).
//
// The memory is independent of any one learner handle (apex.Agent may rebuild its learner for another batch size):
// every call that uses a learner takes it as an argument.  All work of the memory is totally ordered: each call first
// makes the stream it enqueues on wait for `ev_last` (recorded after the previous call's last enqueue, on whichever
// stream that was) and records it again after its own last enqueue.
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "apex_defs.cuh"
#include "replay_tree.cuh"

using namespace drl;

namespace {

// one pinned, device-mapped host block reused call after call; `ev` is recorded after the last device work that reads
// it, and the host waits for it before writing the block again
struct PinnedBlock {
  uint8_t* h = nullptr;
  uint8_t* d = nullptr;           // device alias of h
  size_t bytes = 0;
  cudaEvent_t ev = nullptr;
};

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

struct drl_apex_replay {
  int device = 0;
  int64_t capacity = 0;
  int levels = 0;                      // warps of the tree update kernel
  cudaStream_t stream = nullptr;       // calls that use no learner
  cudaEvent_t ev_last = nullptr;       // after the memory's last enqueue
  double* tree = nullptr;              // [2 * capacity - 1]
  // the transitions, zero-initialised: a leaf past n_entries reached through float drift gathers a defined record
  uint8_t* state = nullptr;            // [capacity][84,84,4]
  uint8_t* next_state = nullptr;       // [capacity][84,84,4]
  int32_t *previous_action = nullptr, *action = nullptr;
  float* reward = nullptr;
  uint8_t* done = nullptr;
  // the last sample, on the device
  int64_t *d_tree_index = nullptr, *d_data_index = nullptr;
  double *d_priority = nullptr, *d_is_weight = nullptr;
  int sample_cap = 0, last_n = 0;
  // ingest: pinned block -> one H2D -> the device block (both of ingest_cap transitions)
  PinnedBlock ingest;
  uint8_t* d_ingest = nullptr;
  int ingest_cap = 0;
  PinnedBlock args;                    // the uniforms / indices / errors of calls without a learner
  std::vector<PinnedBlock> uniforms;   // per learner slot: the uniforms of drl_apex_replay_step_async
  // host-side state of Memory that follows from the call sequence (per.cu keeps the same, in the same types)
  int64_t cursor = 0, n_entries = 0;
  double beta = 0.4;
  std::vector<void*> allocs;
  std::recursive_mutex mu;
};

namespace {

int check_replay(const drl_apex_replay* r) {
  if (!r) { set_error("null apex replay handle"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

void free_pinned(PinnedBlock& b) {
  if (b.ev) cudaEventSynchronize(b.ev);
  if (b.h) cudaFreeHost(b.h);
  b.h = b.d = nullptr;
  b.bytes = 0;
}

// waits until the device no longer reads the block, growing it to `bytes` first if needed
int acquire(PinnedBlock& b, size_t bytes) {
  if (!b.ev) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&b.ev, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventSynchronize(b.ev));
  if (b.bytes < bytes) {
    free_pinned(b);
    DRL_CUDA_CHECK(cudaHostAlloc((void**)&b.h, bytes, cudaHostAllocMapped));
    DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&b.d, b.h, 0));
    b.bytes = bytes;
  }
  return DRL_OK;
}

// device buffers sized for n draws / n ingested transitions; regrowing waits for the memory's earlier work
int ensure_sample(drl_apex_replay* r, int n) {
  if (n <= r->sample_cap) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  for (void* p : {(void*)r->d_tree_index, (void*)r->d_data_index, (void*)r->d_priority, (void*)r->d_is_weight})
    if (p) cudaFree(p);
  r->d_tree_index = r->d_data_index = nullptr;
  r->d_priority = r->d_is_weight = nullptr;
  r->sample_cap = 0;
  DRL_CUDA_CHECK(cudaMalloc(&r->d_tree_index, (size_t)n * 8));
  DRL_CUDA_CHECK(cudaMalloc(&r->d_data_index, (size_t)n * 8));
  DRL_CUDA_CHECK(cudaMalloc(&r->d_priority, (size_t)n * 8));
  DRL_CUDA_CHECK(cudaMalloc(&r->d_is_weight, (size_t)n * 8));
  r->sample_cap = n;
  return DRL_OK;
}

int ensure_ingest(drl_apex_replay* r, int n) {
  DRL_TRY(acquire(r->ingest, IngestLayout(n).bytes));
  if (n <= r->ingest_cap) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  if (r->d_ingest) cudaFree(r->d_ingest);
  r->d_ingest = nullptr;
  r->ingest_cap = 0;
  DRL_CUDA_CHECK(cudaMalloc(&r->d_ingest, IngestLayout(n).bytes));
  r->ingest_cap = n;
  return DRL_OK;
}

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

// the stream of this call, ordered after the memory's previous work
int begin(drl_apex_replay* r, cudaStream_t s) {
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(s, r->ev_last, 0));
  return DRL_OK;
}
int end(drl_apex_replay* r, cudaStream_t s) {
  DRL_CUDA_CHECK(cudaEventRecord(r->ev_last, s));
  return DRL_OK;
}

int launch_update(drl_apex_replay* r, cudaStream_t s, int n, const int64_t* tree_index, int64_t first,
                  const double* err64, const float* err32) {
  prof_mark(s, "replay_tree_update");
  DRL_CUDA_CHECK((launch_k(replay_tree_update_kernel, 1, 32 * r->levels, 0, s, r->tree, r->capacity, n, tree_index,
                           first, err64, err32)));
  return DRL_OK;
}

// Memory.sample's beta step (:395) and the sample kernel over n draws with the uniforms at u01_dev
int launch_sample(drl_apex_replay* r, cudaStream_t s, int n, const double* u01_dev, float* weight32) {
  r->beta = fmin(1.0, r->beta + kReplayBetaInc);
  prof_mark(s, "replay_sample");
  DRL_CUDA_CHECK((launch_k(replay_sample_kernel, 1, 256, 0, s, r->tree, r->capacity, n, u01_dev, (double)r->n_entries,
                           r->beta, r->d_tree_index, r->d_data_index, r->d_priority, r->d_is_weight, weight32)));
  r->last_n = n;
  return DRL_OK;
}

int check_u01(int n, const double* u01) {
  for (int i = 0; i < n; ++i)
    if (!(u01[i] >= 0.0 && u01[i] <= 1.0)) { set_error("apex replay: u01[%d] = %g is not in [0, 1]", i, u01[i]); return DRL_ERR_INVALID; }
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
  if (capacity < 2 || capacity > kReplayMaxCapacity) {
    set_error("apex replay: capacity must be in [2, 2^31] (got %lld)", (long long)capacity);
    return DRL_ERR_INVALID;
  }
  if (device < 0 || drl_device_count() <= device) { set_error("CUDA device %d not available (no CPU fallback)", device); return DRL_ERR_CUDA; }
  drl_apex_replay* r = new drl_apex_replay();
  r->device = device;
  r->capacity = capacity;
  r->levels = replay_tree_levels(capacity);
  int rc = [&]() -> int {
    const size_t C = (size_t)capacity;
    DRL_CUDA_CHECK(cudaSetDevice(device));
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&r->ev_last, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventRecord(r->ev_last, r->stream));
    DRL_TRY(dev_alloc(r, &r->tree, 2 * C - 1));
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
  cudaSetDevice(r->device);
  if (r->ev_last) cudaEventSynchronize(r->ev_last);
  free_pinned(r->ingest);
  free_pinned(r->args);
  for (PinnedBlock& b : r->uniforms) free_pinned(b);
  for (PinnedBlock* b : {&r->ingest, &r->args}) if (b->ev) cudaEventDestroy(b->ev);
  for (PinnedBlock& b : r->uniforms) if (b.ev) cudaEventDestroy(b.ev);
  for (void* p : {(void*)r->d_tree_index, (void*)r->d_data_index, (void*)r->d_priority, (void*)r->d_is_weight,
                  (void*)r->d_ingest})
    if (p) cudaFree(p);
  for (void* p : r->allocs) cudaFree(p);
  if (r->ev_last) cudaEventDestroy(r->ev_last);
  if (r->stream) cudaStreamDestroy(r->stream);
  cudaGetLastError();
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
  DRL_TRY(ensure_ingest(r, n));
  const IngestLayout L(n);
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
  DRL_TRY(begin(r, s));
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
  DRL_TRY(launch_update(r, s, n, nullptr, r->cursor, error ? reinterpret_cast<const double*>(d + L.er) : nullptr,
                        error ? nullptr : learner->td_dev));
  DRL_TRY(end(r, s));
  r->cursor = (r->cursor + n) % r->capacity;                 // SumTree.add (:351-359)
  r->n_entries = std::min<int64_t>(r->capacity, r->n_entries + n);
  return DRL_OK;
}

int drl_apex_replay_step_async(drl_apex_replay* r, drl_apex* learner, int32_t slot, const double* u01) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  DRL_TRY(check_learner(r, learner));
  std::lock_guard<std::recursive_mutex> llk(learner->mu);
  DRL_TRY(check_slot(learner, slot));
  if (!u01) { set_error("apex replay step: null u01"); return DRL_ERR_INVALID; }
  if (r->n_entries < 1) { set_error("apex replay step: the memory is empty"); return DRL_ERR_STATE; }
  const int B = learner->B;
  DRL_TRY(check_u01(B, u01));
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(ensure_sample(r, B));
  if ((int)r->uniforms.size() <= slot) r->uniforms.resize(slot + 1);
  PinnedBlock& ub = r->uniforms[slot];
  DRL_TRY(acquire(ub, (size_t)B * 8));
  memcpy(ub.h, u01, (size_t)B * 8);
  const cudaStream_t s = learner->compute;
  AdamSlot& sl = learner->slots[slot];
  const ApexIn& in = learner->in[slot];
  DRL_TRY(begin(r, s));
  if (sl.has_data) DRL_CUDA_CHECK(cudaStreamWaitEvent(s, sl.staged, 0));   // an earlier drl_apex_stage of the slot
  DRL_TRY(launch_sample(r, s, B, reinterpret_cast<const double*>(ub.d), in.weight));
  DRL_CUDA_CHECK(cudaEventRecord(ub.ev, s));
  prof_mark(s, "replay_gather");
  DRL_CUDA_CHECK((launch_k(apex_replay_gather_kernel, dim3(B, 2), 256, 0, s, r->d_data_index, B, r->state,
                           r->next_state, r->previous_action, r->action, r->reward, r->done, in)));
  DRL_CUDA_CHECK(cudaEventRecord(sl.staged, s));
  sl.has_data = true;
  DRL_TRY(adam_run_step(learner, slot));
  // Memory.update of the sampled leaves with the step's |td| (train_apex.py:153-154), before drl_apex_wait returns
  DRL_TRY(launch_update(r, s, B, r->d_tree_index, 0, nullptr, learner->td_dev));
  DRL_CUDA_CHECK(cudaEventRecord(learner->ev_done, s));
  DRL_TRY(end(r, s));
  return DRL_OK;
}

int drl_apex_replay_sample(drl_apex_replay* r, int32_t n, const double* u01, int64_t* tree_index, int64_t* data_index,
                           double* priority, double* is_weight) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || !u01 || !tree_index || !data_index || !priority || !is_weight) { set_error("apex replay sample: bad argument"); return DRL_ERR_INVALID; }
  if (r->n_entries < 1) { set_error("apex replay sample: the memory is empty"); return DRL_ERR_STATE; }
  DRL_TRY(check_u01(n, u01));
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(ensure_sample(r, n));
  DRL_TRY(acquire(r->args, (size_t)n * 8));
  memcpy(r->args.h, u01, (size_t)n * 8);
  const cudaStream_t s = r->stream;
  DRL_TRY(begin(r, s));
  DRL_TRY(launch_sample(r, s, n, reinterpret_cast<const double*>(r->args.d), nullptr));
  DRL_CUDA_CHECK(cudaEventRecord(r->args.ev, s));
  DRL_TRY(end(r, s));
  DRL_TRY(drl_apex_replay_last_sample(r, tree_index, priority, is_weight));
  DRL_CUDA_CHECK(cudaMemcpy(data_index, r->d_data_index, (size_t)n * 8, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_apex_replay_update(drl_apex_replay* r, int32_t n, const int64_t* tree_index, const double* error) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || !tree_index || !error) { set_error("apex replay update: bad argument"); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i)
    if (tree_index[i] < r->capacity - 1 || tree_index[i] >= 2 * r->capacity - 1) {
      set_error("apex replay update: %lld is not a leaf index", (long long)tree_index[i]);
      return DRL_ERR_INVALID;
    }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(acquire(r->args, (size_t)n * 16));
  memcpy(r->args.h, tree_index, (size_t)n * 8);
  memcpy(r->args.h + (size_t)n * 8, error, (size_t)n * 8);
  const cudaStream_t s = r->stream;
  DRL_TRY(begin(r, s));
  DRL_TRY(launch_update(r, s, n, reinterpret_cast<const int64_t*>(r->args.d), 0,
                        reinterpret_cast<const double*>(r->args.d + (size_t)n * 8), nullptr));
  DRL_CUDA_CHECK(cudaEventRecord(r->args.ev, s));
  return end(r, s);
}

int drl_apex_replay_last_sample(drl_apex_replay* r, int64_t* tree_index, double* priority, double* is_weight) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (r->last_n < 1) { set_error("apex replay last_sample: nothing has been sampled"); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  const size_t bytes = (size_t)r->last_n * 8;
  if (tree_index) DRL_CUDA_CHECK(cudaMemcpy(tree_index, r->d_tree_index, bytes, cudaMemcpyDeviceToHost));
  if (priority) DRL_CUDA_CHECK(cudaMemcpy(priority, r->d_priority, bytes, cudaMemcpyDeviceToHost));
  if (is_weight) DRL_CUDA_CHECK(cudaMemcpy(is_weight, r->d_is_weight, bytes, cudaMemcpyDeviceToHost));
  return DRL_OK;
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

int drl_apex_replay_total(drl_apex_replay* r, double* total) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!total) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  DRL_CUDA_CHECK(cudaMemcpy(total, r->tree, 8, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int drl_apex_replay_size(drl_apex_replay* r, int64_t* n_entries) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!n_entries) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n_entries = r->n_entries;
  return DRL_OK;
}

int drl_apex_replay_beta(drl_apex_replay* r, double* beta) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!beta) { set_error("null argument"); return DRL_ERR_INVALID; }
  *beta = r->beta;
  return DRL_OK;
}

}  // extern "C"
