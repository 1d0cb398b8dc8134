// apex_actor_buffer.cu -- the n LocalBuffers of one Ape-X vector actor in device memory, behind
// drl_apex_actor_buffer_* (include/drl_b200.h; DESIGN.md section 14): buffer_queue.LocalBuffer
// (distributed_queue/buffer_queue.py:274-318) for n environments that append in lockstep, and its sample pushed into a
// device Ape-X queue (drl_apex_queue, traj_queue.cuh) without a host copy.
//
// Storage: n * capacity rows in the replay memory's field layout (state and next_state u8 [84,84,4], previous_action and
// action i32, reward f32, done u8: 56,461 B per row); environment e's ring row r is row e * capacity + r.  One host
// cursor (`appended`) and one length describe every environment's ring: deque index j is ring row
// (appended - len + j) mod capacity, the transition collections.deque(maxlen=capacity) would hold at index j.
//
// Ordering: every append and push runs on the buffer's own stream, so a push's gather reads the rows after the appends
// before it.  A push's gather waits for the queue slot's release event and is followed by the slot's commit event.
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "apex_defs.cuh"
#include "traj_queue.cuh"

using namespace drl;

namespace {

constexpr int kFrame16 = Geo::FRAME / 16;    // 1,764 16-byte vectors per 84x84x4 frame

size_t ab_align(size_t v) { return (v + 255) / 256 * 256; }

// The upload of one append, in the pinned block and in its device copy alike:
// src i32 [n] | previous_action i32 [n] | action i32 [n] | reward f32 [n] | done u8 [n] | next_state [n] frames |
// state [k] frames (only the k rows whose state the device does not hold).  One H2D moves the first `bytes(k)` bytes.
struct UploadLayout {
  size_t src, pa, ac, rw, dn, next, state;
  explicit UploadLayout(size_t n) {
    size_t off = 0;
    src = off; off = ab_align(off + n * 4);
    pa = off; off = ab_align(off + n * 4);
    ac = off; off = ab_align(off + n * 4);
    rw = off; off = ab_align(off + n * 4);
    dn = off; off = ab_align(off + n);
    next = off;
    state = next + n * Geo::FRAME;
  }
  size_t bytes(size_t k) const { return state + k * Geo::FRAME; }
};

}  // namespace

namespace drl {

struct BufferRows {
  uint8_t* state;           // [n * capacity][84,84,4]
  uint8_t* next_state;      // [n * capacity][84,84,4]
  int32_t* previous_action; // [n * capacity]
  int32_t* action;
  float* reward;
  uint8_t* done;
};

struct UploadView {
  const int32_t* src;       // [n]: row i's state is upload state frame src[i], or (-1) the previous row's next_state
  const int32_t* pa;
  const int32_t* ac;
  const float* rw;
  const uint8_t* dn;
  const uint8_t* next;      // [n] frames
  const uint8_t* state;     // [k] frames
};

// the ring rows of one push, by value (T <= kApexQueueMaxT)
struct PushRows {
  int32_t row[kApexQueueMaxT];
};

}  // namespace drl

struct drl_apex_actor_buffer {
  int device = 0, n = 0, A = 0;
  int64_t capacity = 0;
  int64_t appended = 0, len = 0;       // appends so far (every environment), deque length
  bool have_prev = false;              // the pinned block's next_state frames are the device's newest next_state rows
  cudaStream_t stream = nullptr;
  BufferRows rows{};
  UploadLayout lay{0};
  uint8_t* h_up = nullptr;             // pinned upload block
  uint8_t* d_up = nullptr;             // its device copy
  cudaEvent_t ev_up = nullptr;         // after the last H2D that reads h_up
  std::vector<void*> allocs;
  std::mutex mu;
};

namespace drl {

// One append: block (i, 0) writes environment i's state (from the upload, or on the device from the same environment's
// previous next_state row) and the four scalars into ring row `cur`; block (i, 1) writes its next_state.  `prev` is the
// previous ring row; capacity >= 2 keeps it apart from `cur`, so no block reads a row another block writes.
__global__ void __launch_bounds__(256) apex_buffer_append_kernel(const UploadView up, BufferRows rows, int64_t capacity,
                                                                  int64_t cur, int64_t prev) {
  kernel_prologue();
  const int i = blockIdx.x, half = blockIdx.y;
  const int64_t dst_row = (int64_t)i * capacity + cur;
  const uint4* src;
  uint4* dst;
  if (half == 0) {
    const int s = up.src[i];
    src = s >= 0 ? reinterpret_cast<const uint4*>(up.state + (size_t)s * Geo::FRAME)
                 : reinterpret_cast<const uint4*>(rows.next_state + (size_t)((int64_t)i * capacity + prev) * Geo::FRAME);
    dst = reinterpret_cast<uint4*>(rows.state + (size_t)dst_row * Geo::FRAME);
  } else {
    src = reinterpret_cast<const uint4*>(up.next + (size_t)i * Geo::FRAME);
    dst = reinterpret_cast<uint4*>(rows.next_state + (size_t)dst_row * Geo::FRAME);
  }
  for (int k = threadIdx.x; k < kFrame16; k += blockDim.x) dst[k] = src[k];
  if (half == 0 && threadIdx.x == 0) {
    rows.previous_action[dst_row] = up.pa[i];
    rows.action[dst_row] = up.ac[i];
    rows.reward[dst_row] = up.rw[i];
    rows.done[dst_row] = up.dn[i];
  }
}

// One push: the T sampled rows of environment `env` into a queue slot as an ApexIn of n = T rows.  Block (t, 0) copies
// row t's state into frame t and its scalars; block (t, 1) its next_state into frame T + t.
__global__ void __launch_bounds__(256) apex_buffer_push_kernel(const BufferRows rows, int64_t base, const PushRows pr,
                                                                int T, ApexIn out) {
  kernel_prologue();
  const int t = blockIdx.x, half = blockIdx.y;
  const int64_t row = base + pr.row[t];
  const uint4* src = reinterpret_cast<const uint4*>((half ? rows.next_state : rows.state) + (size_t)row * Geo::FRAME);
  uint4* dst = reinterpret_cast<uint4*>(out.frames + ((size_t)half * T + t) * Geo::FRAME);
  for (int k = threadIdx.x; k < kFrame16; k += blockDim.x) dst[k] = src[k];
  if (half == 0 && threadIdx.x == 0) {
    out.pa2[t] = rows.previous_action[row];
    out.pa2[T + t] = rows.action[row];
    out.reward[t] = rows.reward[row];
    out.done[t] = rows.done[row];
  }
}

}  // namespace drl

namespace {

using Lock = std::lock_guard<std::mutex>;

template <class P>
int buf_alloc(drl_apex_actor_buffer* b, P** p, size_t count) {
  DRL_CUDA_CHECK(cudaMalloc((void**)p, count * sizeof(P)));
  b->allocs.push_back(*p);
  DRL_CUDA_CHECK(cudaMemset(*p, 0, count * sizeof(P)));
  return DRL_OK;
}

int check_buffer(const drl_apex_actor_buffer* b) {
  if (!b) { set_error("null apex actor buffer handle"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

}  // namespace

extern "C" {

int drl_apex_actor_buffer_create(int32_t n, int32_t capacity, int32_t num_action, int32_t device,
                                 drl_apex_actor_buffer** out) {
  if (!out) { set_error("null argument"); return DRL_ERR_INVALID; }
  *out = nullptr;
  if (n < 1) { set_error("apex actor buffer: n must be >= 1 (got %d)", n); return DRL_ERR_INVALID; }
  if (capacity < 2) { set_error("apex actor buffer: capacity must be >= 2 (got %d)", capacity); return DRL_ERR_INVALID; }
  if (num_action < 2 || num_action > 32) {
    set_error("apex actor buffer: num_action must be in [2, 32] (got %d)", num_action);
    return DRL_ERR_INVALID;
  }
  if (device < 0 || drl_device_count() <= device) {
    set_error("CUDA device %d not available (no CPU fallback)", device);
    return DRL_ERR_CUDA;
  }
  drl_apex_actor_buffer* b = new drl_apex_actor_buffer();
  b->device = device;
  b->n = n;
  b->A = num_action;
  b->capacity = capacity;
  b->lay = UploadLayout(n);
  const int rc = [&]() -> int {
    const size_t rows = (size_t)n * capacity;
    DRL_CUDA_CHECK(cudaSetDevice(device));
    DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&b->ev_up, cudaEventDisableTiming));
    DRL_TRY(buf_alloc(b, &b->rows.state, rows * Geo::FRAME));
    DRL_TRY(buf_alloc(b, &b->rows.next_state, rows * Geo::FRAME));
    DRL_TRY(buf_alloc(b, &b->rows.previous_action, rows));
    DRL_TRY(buf_alloc(b, &b->rows.action, rows));
    DRL_TRY(buf_alloc(b, &b->rows.reward, rows));
    DRL_TRY(buf_alloc(b, &b->rows.done, rows));
    const size_t up = b->lay.bytes(n);
    DRL_TRY(buf_alloc(b, &b->d_up, up));
    DRL_CUDA_CHECK(cudaMallocHost((void**)&b->h_up, up));
    DRL_CUDA_CHECK(cudaDeviceSynchronize());
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    const std::string keep = get_error();
    drl_apex_actor_buffer_destroy(b);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = b;
  return DRL_OK;
}

int drl_apex_actor_buffer_destroy(drl_apex_actor_buffer* b) {
  if (!b) return DRL_OK;
  cudaSetDevice(b->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  if (b->h_up) cudaFreeHost(b->h_up);
  for (void* p : b->allocs) cudaFree(p);
  if (b->ev_up) cudaEventDestroy(b->ev_up);
  if (b->stream) cudaStreamDestroy(b->stream);
  cudaGetLastError();
  delete b;
  return DRL_OK;
}

int drl_apex_actor_buffer_size(drl_apex_actor_buffer* b, int64_t* len) {
  DRL_TRY(check_buffer(b));
  if (!len) { set_error("apex actor buffer size: null argument"); return DRL_ERR_INVALID; }
  Lock lk(b->mu);
  *len = b->len;
  return DRL_OK;
}

int drl_apex_actor_buffer_append(drl_apex_actor_buffer* b, int32_t n, const uint8_t* state, const uint8_t* next_state,
                                 const int32_t* previous_action, const int32_t* action, const float* reward,
                                 const uint8_t* done) {
  DRL_TRY(check_buffer(b));
  if (!state || !next_state || !previous_action || !action || !reward || !done) {
    set_error("apex actor buffer append: null input pointer");
    return DRL_ERR_INVALID;
  }
  if (n != b->n) { set_error("apex actor buffer append: %d rows, the buffer holds %d environments", n, b->n); return DRL_ERR_INVALID; }
  // the learner's embedding gathers table + action * 256 without a bounds check, and the ingest trusts the queue
  for (int i = 0; i < n; ++i)
    if (previous_action[i] < 0 || previous_action[i] >= b->A || action[i] < 0 || action[i] >= b->A) {
      set_error("apex actor buffer append: an action of environment %d is not in [0, %d)", i, b->A);
      return DRL_ERR_INVALID;
    }
  Lock lk(b->mu);
  NvtxRange nv("drl:apex_actor_buffer_append");
  const UploadLayout& L = b->lay;
  DRL_CUDA_CHECK(cudaSetDevice(b->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(b->ev_up));          // the previous H2D no longer reads the block
  uint8_t* h = b->h_up;
  int32_t* src = reinterpret_cast<int32_t*>(h + L.src);
  // a row's state crosses PCIe only when the device does not hold it as the environment's previous next_state (the
  // first append, and the step after an episode reset); the block still holds the previous append's next_state frames
  int k = 0;
  for (int i = 0; i < n; ++i) {
    const uint8_t* s = state + (size_t)i * Geo::FRAME;
    if (b->have_prev && memcmp(s, h + L.next + (size_t)i * Geo::FRAME, Geo::FRAME) == 0) {
      src[i] = -1;
    } else {
      memcpy(h + L.state + (size_t)k * Geo::FRAME, s, Geo::FRAME);
      src[i] = k++;
    }
  }
  b->have_prev = false;                                    // until this append is enqueued whole
  memcpy(h + L.next, next_state, (size_t)n * Geo::FRAME);
  memcpy(h + L.pa, previous_action, (size_t)n * 4);
  memcpy(h + L.ac, action, (size_t)n * 4);
  memcpy(h + L.rw, reward, (size_t)n * 4);
  memcpy(h + L.dn, done, (size_t)n);
  const cudaStream_t s = b->stream;
  uint8_t* d = b->d_up;
  DRL_CUDA_CHECK(cudaMemcpyAsync(d, h, L.bytes(k), cudaMemcpyHostToDevice, s));
  DRL_CUDA_CHECK(cudaEventRecord(b->ev_up, s));
  const UploadView up{reinterpret_cast<const int32_t*>(d + L.src), reinterpret_cast<const int32_t*>(d + L.pa),
                      reinterpret_cast<const int32_t*>(d + L.ac),  reinterpret_cast<const float*>(d + L.rw),
                      d + L.dn, d + L.next, d + L.state};
  const int64_t cur = b->appended % b->capacity, prev = (b->appended + b->capacity - 1) % b->capacity;
  DRL_CUDA_CHECK((launch_k(apex_buffer_append_kernel, dim3(n, 2), 256, 0, s, up, b->rows, b->capacity, cur, prev)));
  b->appended++;
  if (b->len < b->capacity) b->len++;
  b->have_prev = true;
  return DRL_OK;
}

int drl_apex_actor_buffer_push(drl_apex_actor_buffer* b, drl_apex_queue* q, int32_t env, const int32_t* order,
                               int32_t timeout_ms) {
  DRL_TRY(check_buffer(b));
  if (!q) { set_error("null apex queue handle"); return DRL_ERR_INVALID; }
  if (!order) { set_error("apex actor buffer push: null order"); return DRL_ERR_INVALID; }
  if (q->device != b->device) {
    set_error("apex actor buffer push: the queue is on device %d, the buffer on device %d", q->device, b->device);
    return DRL_ERR_INVALID;
  }
  if (q->A != b->A) {
    set_error("apex actor buffer push: the queue has num_action %d, the buffer %d", q->A, b->A);
    return DRL_ERR_INVALID;
  }
  if (env < 0 || env >= b->n) { set_error("apex actor buffer push: env = %d is outside [0, %d)", env, b->n); return DRL_ERR_INVALID; }
  const int T = q->T;
  {
    Lock lk(b->mu);
    for (int t = 0; t < T; ++t)
      if (order[t] < 0 || order[t] >= b->len) {
        set_error("apex actor buffer push: order[%d] = %d is outside [0, %lld) (the buffer's length)", t, order[t],
                  (long long)b->len);
        return DRL_ERR_INVALID;
      }
  }
  // reserve without the buffer's lock, blocking while the queue is full; the length only grows meanwhile, so the
  // indices checked above stay valid
  std::vector<TrajSegment> segs;
  DRL_TRY(traj_queue_reserve(q, 1, timeout_ms, &segs));
  Lock lk(b->mu);
  NvtxRange nv("drl:apex_actor_buffer_push");
  const TrajSegment& g = segs[0];
  const int rc = [&]() -> int {
    PushRows pr;
    for (int t = 0; t < T; ++t) pr.row[t] = (int32_t)((b->appended - b->len + order[t]) % b->capacity);
    const ApexIn slot{q->field(g.slot, kApexQFrames), reinterpret_cast<int32_t*>(q->field(g.slot, kApexQPa2)),
                      reinterpret_cast<float*>(q->field(g.slot, kApexQReward)), q->field(g.slot, kApexQDone), nullptr};
    const cudaStream_t s = b->stream;
    DRL_CUDA_CHECK(cudaSetDevice(b->device));
    DRL_CUDA_CHECK(cudaStreamWaitEvent(s, g.ev_release, 0));
    DRL_CUDA_CHECK((launch_k(apex_buffer_push_kernel, dim3(T, 2), 256, 0, s, b->rows, (int64_t)env * b->capacity, pr,
                             T, slot)));
    DRL_CUDA_CHECK(cudaEventRecord(g.ev_commit, s));
    return DRL_OK;
  }();
  if (rc != DRL_OK) {
    // the reserved position will never be filled: the queue goes into its failed state instead of blocking its
    // consumer forever (as a recorder's commit does)
    traj_queue_fail(q, get_error());
    return rc;
  }
  traj_queue_commit(q, segs);
  return DRL_OK;
}

int drl_apex_actor_buffer_read(drl_apex_actor_buffer* b, int32_t env, int64_t j, uint8_t* state, uint8_t* next_state,
                               int32_t* previous_action, int32_t* action, float* reward, uint8_t* done) {
  DRL_TRY(check_buffer(b));
  if (!state || !next_state || !previous_action || !action || !reward || !done) {
    set_error("apex actor buffer read: null output pointer");
    return DRL_ERR_INVALID;
  }
  Lock lk(b->mu);
  if (env < 0 || env >= b->n || j < 0 || j >= b->len) {
    set_error("apex actor buffer read: (env %d, index %lld) is outside [0, %d) x [0, %lld)", env, (long long)j, b->n,
              (long long)b->len);
    return DRL_ERR_INVALID;
  }
  DRL_CUDA_CHECK(cudaSetDevice(b->device));
  DRL_CUDA_CHECK(cudaStreamSynchronize(b->stream));
  const size_t row = (size_t)env * b->capacity + (size_t)((b->appended - b->len + j) % b->capacity);
  auto cp = [](void* dst, const void* src, size_t bytes) { return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost); };
  DRL_CUDA_CHECK(cp(state, b->rows.state + row * Geo::FRAME, Geo::FRAME));
  DRL_CUDA_CHECK(cp(next_state, b->rows.next_state + row * Geo::FRAME, Geo::FRAME));
  DRL_CUDA_CHECK(cp(previous_action, b->rows.previous_action + row, 4));
  DRL_CUDA_CHECK(cp(action, b->rows.action + row, 4));
  DRL_CUDA_CHECK(cp(reward, b->rows.reward + row, 4));
  DRL_CUDA_CHECK(cp(done, b->rows.done + row, 1));
  return DRL_OK;
}

}  // extern "C"
