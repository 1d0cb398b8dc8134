// r2d2_replay.cu -- the R2D2 prioritized sequence replay memory on the device, behind drl_r2d2_replay_*
// (include/drl_b200.h): buffer_queue.Memory (distributed_queue/buffer_queue.py:371-415) with one stored-state sequence
// per record in HBM, its sum tree on the device, and the learner loop of train_r2d2.py:87-165 -- ingest with the
// learner's batched |td|, stratified sample, minibatch gather into a learner staging slot, step, priority update -- as
// kernels on the learner's compute stream, without a host round trip between steps (DESIGN.md section 11).  This file
// holds what depends on one record being a sequence: the storage, the sequence store and gather kernels and the ingest
// layout; the sum tree, the ordering of the memory's work and the sample / update / total / size / beta bodies are the
// shared core's (replay_core.cuh).
//
// A record keeps only step 0 of the stored (h, c): agent/r2d2.py:110-111 and :135-136 feed h[:, 0] / c[:, 0] of the
// stored [S, L] states, and nothing reads the other steps.  The memory is independent of any one learner handle
// (r2d2.Agent may rebuild its learner for another batch size): every call that uses a learner takes it as an argument.
#include <string.h>

#include <mutex>
#include <string>

#include "r2d2_defs.cuh"
#include "replay_core.cuh"
#include "traj_queue.cuh"

using namespace drl;

namespace drl {

// Batch-major sequence rows: the memory's storage (rows = capacity) and a learner slot's R2In views (rows = B) share
// this layout, so one row is one contiguous run of each field.
struct R2SeqRows {
  uint8_t* frames;         // [rows, S, 84, 84, C]
  int32_t* pa;             // [rows, S]
  int32_t* action;         // [rows, S]
  float* h0;               // [rows, L]
  float* c0;               // [rows, L]
  float* reward;           // [rows, S]
  uint8_t* done;           // [rows, S]
};

// Block (i, t) copies frame t of row src_row into row dst_row as 16-byte vectors (frame16 = 84 * 84 * C / 16 of them:
// 441 or 1,764), and thread 0 the step's four scalars; block (i, 0) also copies the row's h0 and c0 (L / 4 vectors each,
// L = lstm_size).
__device__ __forceinline__ void copy_seq_step(const R2SeqRows& src, int64_t src_row, const R2SeqRows& dst,
                                              int64_t dst_row, int S, int frame16, int L) {
  const int t = blockIdx.y;
  const size_t fs = ((size_t)src_row * S + t) * frame16, fd = ((size_t)dst_row * S + t) * frame16;
  const uint4* __restrict__ s4 = reinterpret_cast<const uint4*>(src.frames) + fs;
  uint4* __restrict__ d4 = reinterpret_cast<uint4*>(dst.frames) + fd;
  for (int k = threadIdx.x; k < frame16; k += blockDim.x) d4[k] = s4[k];
  if (threadIdx.x == 0) {
    const size_t so = (size_t)src_row * S + t, dof = (size_t)dst_row * S + t;
    dst.pa[dof] = src.pa[so];
    dst.action[dof] = src.action[so];
    dst.reward[dof] = src.reward[so];
    dst.done[dof] = src.done[so];
  }
  if (t == 0)
    for (int i = threadIdx.x; i < 2 * (L / 4); i += blockDim.x) {
      const int k = i % (L / 4);
      const float* s = i < L / 4 ? src.h0 : src.c0;
      float* d = i < L / 4 ? dst.h0 : dst.c0;
      reinterpret_cast<float4*>(d + (size_t)dst_row * L)[k] = reinterpret_cast<const float4*>(s + (size_t)src_row * L)[k];
    }
}

// Ingest: the n sequences of the ingest block (rows 0..n-1) into the storage rows (first + i) mod capacity.  Grid (n, S).
__global__ void __launch_bounds__(256) replay_store_seq_kernel(const R2SeqRows in, int64_t first, int64_t capacity,
                                                                const R2SeqRows mem, int S, int frame16, int L) {
  kernel_prologue();
  copy_seq_step(in, blockIdx.x, mem, (first + blockIdx.x) % capacity, S, frame16, L);
}

// The minibatch of a training step: the sampled storage rows data_index[0, B) into a learner slot's views (rows 0..B-1),
// in the layout drl_r2d2_stage writes.  The importance weights are written by the sample kernel.  Grid (B, S).
__global__ void __launch_bounds__(256) replay_gather_seq_kernel(const int64_t* __restrict__ data_index,
                                                                 const R2SeqRows mem, const R2SeqRows out, int S,
                                                                 int frame16, int L) {
  kernel_prologue();
  copy_seq_step(mem, data_index[blockIdx.x], out, blockIdx.x, S, frame16, L);
}

}  // namespace drl

namespace {

constexpr const char* kName = "r2d2 replay";

// device ingest block of n sequences, laid out as an R2In of n rows:
// frames [n,S] | pa [n,S] | action [n,S] | h0 [n,L] | c0 [n,L] | reward [n,S] | done [n,S] | error [n] (double, the
// caller's priorities when given)
struct IngestLayout {
  size_t fr, pa, ac, h, c, rw, dn, er, bytes;
  IngestLayout(size_t n, size_t S, size_t frame, size_t L) {
    size_t off = 0;
    fr = off; off = align_up(off + n * S * frame, 256);
    pa = off; off = align_up(off + n * S * 4, 256);
    ac = off; off = align_up(off + n * S * 4, 256);
    h = off; off = align_up(off + n * L * 4, 256);
    c = off; off = align_up(off + n * L * 4, 256);
    rw = off; off = align_up(off + n * S * 4, 256);
    dn = off; off = align_up(off + n * S, 256);
    er = off; off = align_up(off + n * 8, 256);
    bytes = off;
  }
};

}  // namespace

// the sum tree, the ordering and the sample / update state are the shared core's (replay_core.cuh)
struct drl_r2d2_replay : ReplayCore {
  int S = 0, C = 1, A = 0, L = kR2L;    // L: lstm_size, the width of a record's h0 / c0
  size_t frame = 0;                    // bytes of one 84x84xC frame
  // the sequences, zero-initialised: a leaf past n_entries reached through float drift gathers a defined record
  R2SeqRows mem{};
};

namespace {

int check_replay(const drl_r2d2_replay* r) { return replay_check(r, kName); }

// a learner argument: an R2D2 handle on the memory's device whose sequences and network match the memory's
int check_learner(const drl_r2d2_replay* r, const drl_r2d2* h) {
  DRL_TRY(check_handle(h, "r2d2"));
  if (h->device != r->device) {
    set_error("r2d2 replay: the learner is on device %d, the memory on device %d", h->device, r->device);
    return DRL_ERR_INVALID;
  }
  if (h->S != r->S || h->C != r->C || h->A != r->A || h->L != r->L) {
    set_error("r2d2 replay: the learner has seq_len %d, %d channels, num_action %d and lstm_size %d, the memory %d, %d, "
              "%d and %d", h->S, h->C, h->A, h->L, r->S, r->C, r->A, r->L);
    return DRL_ERR_INVALID;
  }
  return DRL_OK;
}

R2SeqRows slot_rows(const R2In& in) {
  return R2SeqRows{const_cast<uint8_t*>(in.frames), const_cast<int32_t*>(in.pa), const_cast<int32_t*>(in.action),
                   const_cast<float*>(in.h0),       const_cast<float*>(in.c0),   const_cast<float*>(in.reward),
                   const_cast<uint8_t*>(in.done)};
}

}  // namespace

extern "C" {

int drl_r2d2_replay_create(int32_t device, int64_t capacity, int32_t seq_len, int32_t channels, int32_t num_action,
                           drl_r2d2_replay** out) {
  return drl_r2d2_replay_create_lstm(device, capacity, seq_len, channels, num_action, kR2L, out);
}

int drl_r2d2_replay_create_lstm(int32_t device, int64_t capacity, int32_t seq_len, int32_t channels, int32_t num_action,
                                int32_t lstm_size, drl_r2d2_replay** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (lstm_size != kR2L && lstm_size != 256 && lstm_size != 512) {
    set_error("r2d2 replay: lstm_size must be 64, 256 or 512 (got %d)", lstm_size);
    return DRL_ERR_INVALID;
  }
  if (seq_len < 2) { set_error("r2d2 replay: seq_len must be >= 2 (got %d)", seq_len); return DRL_ERR_INVALID; }
  if (channels != 1 && channels != 4) { set_error("r2d2 replay: channels must be 1 or 4 (got %d)", channels); return DRL_ERR_INVALID; }
  if (num_action < 2 || num_action > 32) { set_error("r2d2 replay: num_action must be in [2, 32] (got %d)", num_action); return DRL_ERR_INVALID; }
  DRL_TRY(replay_check_create(kName, device, capacity));
  drl_r2d2_replay* r = new drl_r2d2_replay();
  r->family = kName;
  r->S = seq_len;
  r->C = channels;
  r->A = num_action;
  r->L = lstm_size;
  r->frame = (size_t)Geo::IH * Geo::IW * channels;
  int rc = [&]() -> int {
    const size_t C = (size_t)capacity, S = (size_t)seq_len;
    DRL_TRY(replay_core_init(r, device, capacity));
    R2SeqRows& m = r->mem;
    DRL_TRY(dev_alloc(r, &m.frames, C * S * r->frame));
    DRL_TRY(dev_alloc(r, &m.pa, C * S));
    DRL_TRY(dev_alloc(r, &m.action, C * S));
    DRL_TRY(dev_alloc(r, &m.h0, C * lstm_size));
    DRL_TRY(dev_alloc(r, &m.c0, C * lstm_size));
    DRL_TRY(dev_alloc(r, &m.reward, C * S));
    DRL_TRY(dev_alloc(r, &m.done, C * S));
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    std::string keep = get_error();
    drl_r2d2_replay_destroy(r);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = r;
  return DRL_OK;
}

int drl_r2d2_replay_destroy(drl_r2d2_replay* r) {
  if (!r) return DRL_OK;
  replay_core_release(r);
  delete r;
  return DRL_OK;
}

int drl_r2d2_replay_add(drl_r2d2_replay* r, drl_r2d2* learner, int32_t n, const uint8_t* state,
                        const int32_t* previous_action, const int32_t* action, const float* h0, const float* c0,
                        const float* reward, const uint8_t* done, const double* error) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!state || !previous_action || !action || !h0 || !c0 || !reward || !done) { set_error("r2d2 replay add: null input pointer"); return DRL_ERR_INVALID; }
  if (n < 1 || n > r->capacity) { set_error("r2d2 replay add: n must be in [1, capacity = %lld]", (long long)r->capacity); return DRL_ERR_INVALID; }
  if (!error && !learner) { set_error("r2d2 replay add: without errors the learner computes them (null learner)"); return DRL_ERR_INVALID; }
  std::unique_lock<std::recursive_mutex> llk;
  if (learner) {
    DRL_TRY(check_learner(r, learner));
    llk = std::unique_lock<std::recursive_mutex>(learner->mu);
    if (n > learner->B) { set_error("r2d2 replay add: n = %d exceeds the learner's batch %d", n, learner->B); return DRL_ERR_INVALID; }
  }
  // the embedding gathers table + previous_action * 256 without a bounds check, at ingest and at every later step
  const int S = r->S;
  for (size_t i = 0; i < (size_t)n * S; ++i)
    if (previous_action[i] < 0 || previous_action[i] >= r->A || action[i] < 0 || action[i] >= r->A) {
      set_error("r2d2 replay add: an action of sequence %d, step %d is not in [0, %d)", (int)(i / S), (int)(i % S), r->A);
      return DRL_ERR_INVALID;
    }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  const IngestLayout L(n, S, r->frame, r->L);
  DRL_TRY(replay_ensure_ingest(r, L.bytes));
  uint8_t* h = r->ingest.h;
  const size_t ns = (size_t)n * S;
  memcpy(h + L.fr, state, ns * r->frame);
  memcpy(h + L.pa, previous_action, ns * 4);
  memcpy(h + L.ac, action, ns * 4);
  memcpy(h + L.h, h0, (size_t)n * r->L * 4);
  memcpy(h + L.c, c0, (size_t)n * r->L * 4);
  memcpy(h + L.rw, reward, ns * 4);
  memcpy(h + L.dn, done, ns);
  if (error) memcpy(h + L.er, error, (size_t)n * 8);
  uint8_t* d = r->d_ingest;
  const R2SeqRows rows{d + L.fr, reinterpret_cast<int32_t*>(d + L.pa), reinterpret_cast<int32_t*>(d + L.ac),
                       reinterpret_cast<float*>(d + L.h), reinterpret_cast<float*>(d + L.c),
                       reinterpret_cast<float*>(d + L.rw), d + L.dn};
  const cudaStream_t s = learner ? learner->compute : r->stream;
  DRL_TRY(replay_begin(r, s));
  DRL_CUDA_CHECK(cudaMemcpyAsync(d, h, L.bytes, cudaMemcpyHostToDevice, s));
  DRL_CUDA_CHECK(cudaEventRecord(r->ingest.ev, s));
  if (!error) {
    // agent/r2d2.py:97-130 for all n sequences in one pass: both unrolls + the TD kernel, |td| stays in td_dev
    const R2In in{rows.frames, rows.pa, rows.action, rows.h0, rows.c0, rows.reward, rows.done, nullptr};
    DRL_TRY(enqueue_forward_td(learner, in, n, false, nullptr, nullptr));
    learner->last_n = n;
  }
  prof_mark(s, "replay_store_seq");
  DRL_CUDA_CHECK((launch_k(replay_store_seq_kernel, dim3(n, S), 256, 0, s, rows, r->cursor, r->capacity, r->mem, S,
                           (int)(r->frame / 16), r->L)));
  DRL_TRY(replay_launch_update(r, s, n, nullptr, r->cursor, error ? reinterpret_cast<const double*>(d + L.er) : nullptr,
                               error ? nullptr : learner->td_dev));
  DRL_TRY(replay_end(r, s));
  replay_advance(r, n);
  return DRL_OK;
}

int drl_r2d2_replay_add_from_queue(drl_r2d2_replay* r, drl_r2d2* learner, drl_r2d2_queue* q, int32_t timeout_ms) {
  DRL_TRY(check_replay(r));
  if (!q) { set_error("null r2d2 queue handle"); return DRL_ERR_INVALID; }
  {
    std::lock_guard<std::recursive_mutex> lk(r->mu);
    DRL_TRY(check_learner(r, learner));
    std::lock_guard<std::recursive_mutex> llk(learner->mu);
    if (q->device != r->device) {
      set_error("r2d2 replay add_from_queue: the queue is on device %d, the memory on device %d", q->device, r->device);
      return DRL_ERR_INVALID;
    }
    if (q->S != r->S || q->C != r->C || q->A != r->A) {
      set_error("r2d2 replay add_from_queue: the queue has seq_len %d, %d channels and num_action %d, the memory %d, %d "
                "and %d", q->S, q->C, q->A, r->S, r->C, r->A);
      return DRL_ERR_INVALID;
    }
    if (r->L != kR2L) {
      set_error("r2d2 replay add_from_queue: the queue stores lstm_size %d states, the memory %d", kR2L, r->L);
      return DRL_ERR_INVALID;
    }
    if (q->batch > learner->B) {
      set_error("r2d2 replay add_from_queue: the queue's batch %d exceeds the learner's batch %d", q->batch, learner->B);
      return DRL_ERR_INVALID;
    }
  }
  // wait for a full batch without either lock: actor threads sync their engines from this learner meanwhile
  int qs = 0;
  std::vector<cudaEvent_t> ev_commit;
  DRL_TRY(traj_queue_pop(q, timeout_ms, &qs, &ev_commit));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  std::lock_guard<std::recursive_mutex> llk(learner->mu);
  NvtxRange nv("drl:r2d2_replay_add_from_queue");
  const int n = q->batch, S = r->S;
  const cudaStream_t s = learner->compute;
  // The slot is an R2In of n rows as it is: the learner and the store read it in place.  Unlike drl_r2d2_replay_add,
  // nothing here checks the actions on the host: the queue's only producers are R2D2 recorders, whose acts check every
  // previous action and explore action before recording it, so every recorded action and previous action is in [0, A)
  // (the embedding gathers table + action * 256 without a bounds check).
  const R2SeqRows rows{q->field(qs, kR2QFrames), reinterpret_cast<int32_t*>(q->field(qs, kR2QPa)),
                       reinterpret_cast<int32_t*>(q->field(qs, kR2QAction)), reinterpret_cast<float*>(q->field(qs, kR2QH)),
                       reinterpret_cast<float*>(q->field(qs, kR2QC)), reinterpret_cast<float*>(q->field(qs, kR2QReward)),
                       q->field(qs, kR2QDone)};
  const int rc = [&]() -> int {
    DRL_CUDA_CHECK(cudaSetDevice(r->device));
    DRL_TRY(replay_begin(r, s));
    for (cudaEvent_t e : ev_commit) DRL_CUDA_CHECK(cudaStreamWaitEvent(s, e, 0));
    const R2In in{rows.frames, rows.pa, rows.action, rows.h0, rows.c0, rows.reward, rows.done, nullptr};
    DRL_TRY(enqueue_forward_td(learner, in, n, false, nullptr, nullptr));
    learner->last_n = n;
    prof_mark(s, "replay_store_seq");
    DRL_CUDA_CHECK((launch_k(replay_store_seq_kernel, dim3(n, S), 256, 0, s, rows, r->cursor, r->capacity, r->mem, S,
                             (int)(r->frame / 16), r->L)));
    return replay_launch_update(r, s, n, nullptr, r->cursor, nullptr, learner->td_dev);
  }();
  // the queue slot goes back to the producers either way (their copies into it wait for its release event)
  const int rc_release = traj_queue_release(q, qs, s);
  DRL_TRY(rc);
  DRL_TRY(rc_release);
  DRL_TRY(replay_end(r, s));
  replay_advance(r, n);
  return DRL_OK;
}

int drl_r2d2_replay_step_async(drl_r2d2_replay* r, drl_r2d2* learner, int32_t slot, const double* u01) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  DRL_TRY(check_learner(r, learner));
  std::lock_guard<std::recursive_mutex> llk(learner->mu);
  DRL_TRY(check_slot(learner, slot));
  const int B = learner->B;
  const R2In& in = learner->in[slot];
  const R2SeqRows out = slot_rows(in);
  // Memory.sample -> the minibatch lists and np.stack -> train -> Memory.update with the step's |td|
  // (train_r2d2.py:122-162)
  return replay_step(r, learner, slot, u01, const_cast<float*>(in.weight), learner->td_dev, [&](cudaStream_t s) -> int {
    prof_mark(s, "replay_gather_seq");
    DRL_CUDA_CHECK((launch_k(replay_gather_seq_kernel, dim3(B, r->S), 256, 0, s, r->d_data_index, r->mem, out, r->S,
                             (int)(r->frame / 16), r->L)));
    return DRL_OK;
  });
}

int drl_r2d2_replay_sample(drl_r2d2_replay* r, int32_t n, const double* u01, int64_t* tree_index, int64_t* data_index,
                           double* priority, double* is_weight) {
  return replay_sample(r, kName, n, u01, tree_index, data_index, priority, is_weight);
}

int drl_r2d2_replay_update(drl_r2d2_replay* r, int32_t n, const int64_t* tree_index, const double* error) {
  return replay_update(r, kName, n, tree_index, error);
}

int drl_r2d2_replay_last_sample(drl_r2d2_replay* r, int64_t* tree_index, double* priority, double* is_weight) {
  return replay_last_sample(r, kName, tree_index, priority, is_weight);
}

int drl_r2d2_replay_read(drl_r2d2_replay* r, int64_t data_index, int32_t n, uint8_t* state, int32_t* previous_action,
                         int32_t* action, float* h0, float* c0, float* reward, uint8_t* done) {
  DRL_TRY(check_replay(r));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || data_index < 0 || data_index + n > r->capacity) {
    set_error("r2d2 replay read: rows [%lld, %lld) are not inside [0, %lld)", (long long)data_index,
              (long long)(data_index + n), (long long)r->capacity);
    return DRL_ERR_INVALID;
  }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  const size_t i = (size_t)data_index, m = (size_t)n, S = (size_t)r->S;
  const R2SeqRows& mem = r->mem;
  auto cp = [](void* dst, const void* src, size_t bytes) { return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost); };
  if (state) DRL_CUDA_CHECK(cp(state, mem.frames + i * S * r->frame, m * S * r->frame));
  if (previous_action) DRL_CUDA_CHECK(cp(previous_action, mem.pa + i * S, m * S * 4));
  if (action) DRL_CUDA_CHECK(cp(action, mem.action + i * S, m * S * 4));
  const size_t L = (size_t)r->L;
  if (h0) DRL_CUDA_CHECK(cp(h0, mem.h0 + i * L, m * L * 4));
  if (c0) DRL_CUDA_CHECK(cp(c0, mem.c0 + i * L, m * L * 4));
  if (reward) DRL_CUDA_CHECK(cp(reward, mem.reward + i * S, m * S * 4));
  if (done) DRL_CUDA_CHECK(cp(done, mem.done + i * S, m * S));
  return DRL_OK;
}

int drl_r2d2_replay_total(drl_r2d2_replay* r, double* total) { return replay_total(r, kName, total); }
int drl_r2d2_replay_size(drl_r2d2_replay* r, int64_t* n_entries) { return replay_size(r, kName, n_entries); }
int drl_r2d2_replay_beta(drl_r2d2_replay* r, double* beta) { return replay_beta(r, kName, beta); }

}  // extern "C"
