// replay_core.cu -- the record-independent core of the device replay memories (replay_core.cuh, DESIGN.md sections 10
// and 11): the device sum tree and its two kernels, with the arithmetic of the host tree (per.cu) and the reference's
// Memory (distributed_queue/buffer_queue.py:371-415), the ordering of a memory's work and the C-ABI bodies shared by
// drl_apex_replay_* (apex_replay.cu) and drl_r2d2_replay_* (r2d2_replay.cu).  The tree kernels live in this one
// translation unit: the library is linked without relocatable device code, so a __global__ defined in a header that
// two .cu files include would be defined twice.
#include <string.h>

#include "replay_core.cuh"

namespace drl {

// depth of node x (root 0): floor(log2(x + 1))
__device__ __forceinline__ int tree_depth(int64_t x) { return 63 - __clzll((unsigned long long)(x + 1)); }

// number of levels above the deepest leaf = depth(2 * capacity - 2): the warps of replay_tree_update_kernel
static int replay_tree_levels(int64_t capacity) {
  int d = 0;
  for (unsigned long long v = (unsigned long long)(2 * capacity - 1); v > 1; v >>= 1) ++d;
  return d;
}

// ------------------------------------------------------------------------------------------
// Ordered batch update (Memory.add / Memory.update, :386-388 and :413-415, through SumTree.update / _propagate): for
// i = 0 .. n-1 in order, with leaf_i = tree_index[i] (or capacity - 1 + (first + i) mod capacity when tree_index is
// null) and error_i = err64[i] (or err32[i] when err64 is null):
//   p = pow(error_i + e, a);  change = p - tree[leaf_i];  tree[leaf_i] = p;  tree[ancestor] += change, bottom-up.
// Every node receives its adds in the order of the updates, so the result is the reference's to the last bit for the
// same p.  One block of 32 * levels threads, 32 updates per round:
//   1. thread i of the round computes p_i and change_i; a leaf repeated in the round sees the p of its previous update
//      (the value that update stored), otherwise the tree's value;
//   2. warp d takes the level-d ancestor of each of the 32 leaves, loads them all at once, and lane 0 chains the adds
//      in update order in registers / shared memory (updates that share the node continue from the previous sum);
//      the last update of each node stores it, the last update of each leaf stores p.
// Different levels never share a node, so the warps run in parallel; rounds are separated by __syncthreads.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) replay_tree_update_kernel(double* __restrict__ tree, int64_t capacity, int n,
                                                                   const int64_t* __restrict__ tree_index,
                                                                   int64_t first, const double* __restrict__ err64,
                                                                   const float* __restrict__ err32) {
  kernel_prologue();
  __shared__ int64_t leaf[32];
  __shared__ double pr[32], change[32];
  __shared__ double val[32][33];
  __shared__ int prev_of[32][32];    // latest earlier update of the round on the same node, or -1
  const int lane = threadIdx.x & 31, d = threadIdx.x >> 5;
  for (int base = 0; base < n; base += 32) {
    const int cn = min(32, n - base);
    if (threadIdx.x < cn) {
      const int i = base + threadIdx.x;
      leaf[threadIdx.x] = tree_index ? tree_index[i] : capacity - 1 + (first + i) % capacity;
      const double err = err64 ? err64[i] : (double)err32[i];
      pr[threadIdx.x] = pow(__dadd_rn(err, kReplayE), kReplayA);
    }
    __syncthreads();
    if (threadIdx.x < cn) {
      const int64_t x = leaf[threadIdx.x];
      double prev = tree[x];
      for (int j = (int)threadIdx.x - 1; j >= 0; --j)
        if (leaf[j] == x) { prev = pr[j]; break; }
      change[threadIdx.x] = __dsub_rn(pr[threadIdx.x], prev);
    }
    __syncthreads();
    // warp d: the level-d node on the path of update `lane` (-1 when the leaf is at level d or above)
    int64_t node = -1;
    if (lane < cn) {
      const int64_t x = leaf[lane];
      const int D = tree_depth(x);
      if (d < D) node = ((x + 1) >> (D - d)) - 1;
    }
    const unsigned same = __match_any_sync(0xffffffffu, (long long)node);
    const unsigned before = same & ((1u << lane) - 1u);
    const bool last = (same >> lane) == 1u;               // no later update of this round shares the node
    val[d][lane] = node >= 0 ? tree[node] : 0.0;          // all loads of the level in flight together
    prev_of[d][lane] = before ? 31 - __clz((int)before) : -1;
    __syncwarp();
    if (lane == 0) {                                      // the chain, in update order
      for (int i = 0; i < cn; ++i) {
        const int j = prev_of[d][i];
        val[d][i] = __dadd_rn(j >= 0 ? val[d][j] : val[d][i], change[i]);
      }
    }
    __syncwarp();
    if (node >= 0 && last) tree[node] = val[d][lane];
    if (d == 0 && lane < cn) {
      bool last_leaf = true;
      for (int j = lane + 1; j < cn; ++j)
        if (leaf[j] == leaf[lane]) { last_leaf = false; break; }
      if (last_leaf) tree[leaf[lane]] = pr[lane];
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// Stratified sample (Memory.sample, :390-411, with SumTree.get / _retrieve, :340-347, 366-369), one block, thread i
// per stratum: segment = total / n, s = a + (b - a) u[i] with a = segment i, b = segment (i + 1) -- every product and
// sum rounded on its own (__dmul_rn / __dadd_rn), as the host's unfused code and random.uniform compute them -- then
// the walk from the root with s <= tree[left].  Outputs tree index, data index and priority of each draw and the
// importance weight (n_entries * p / total) ** -beta / max, in double and, when weight32 is not null, as float32.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) replay_sample_kernel(const double* __restrict__ tree, int64_t capacity, int n,
                                                             const double* __restrict__ u01, double n_entries,
                                                             double beta, int64_t* __restrict__ tree_index,
                                                             int64_t* __restrict__ data_index,
                                                             double* __restrict__ priority,
                                                             double* __restrict__ is_weight,
                                                             float* __restrict__ weight32) {
  kernel_prologue();
  __shared__ double red[8];
  const double total = tree[0];
  const double segment = __ddiv_rn(total, (double)n);
  const int64_t len = 2 * capacity - 1;
  double mx = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double a = __dmul_rn(segment, (double)i), b = __dmul_rn(segment, (double)(i + 1));
    double s = __dadd_rn(a, __dmul_rn(__dsub_rn(b, a), u01[i]));
    int64_t idx = 0;
    for (;;) {
      const int64_t left = 2 * idx + 1;
      if (left >= len) break;
      const double tl = tree[left];
      if (s <= tl) {
        idx = left;
      } else {
        s = __dsub_rn(s, tl);
        idx = left + 1;
      }
    }
    const double p = tree[idx];
    tree_index[i] = idx;
    data_index[i] = idx - capacity + 1;
    priority[i] = p;
    const double w = pow(__dmul_rn(n_entries, __ddiv_rn(p, total)), -beta);
    is_weight[i] = w;
    mx = fmax(mx, w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int k = 1; k < (int)(blockDim.x >> 5); ++k) mx = fmax(mx, red[k]);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double w = __ddiv_rn(is_weight[i], mx);
    is_weight[i] = w;
    if (weight32) weight32[i] = __double2float_rn(w);
  }
}

namespace {

void free_pinned(PinnedBlock& b) {
  if (b.ev) cudaEventSynchronize(b.ev);
  if (b.h) cudaFreeHost(b.h);
  b.h = b.d = nullptr;
  b.bytes = 0;
}

}  // namespace

int replay_check(const ReplayCore* r, const char* family) {
  if (!r) { set_error("null %s handle", family); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int replay_check_create(const char* family, int32_t device, int64_t capacity) {
  if (capacity < 2 || capacity > kReplayMaxCapacity) {
    set_error("%s: capacity must be in [2, 2^31] (got %lld)", family, (long long)capacity);
    return DRL_ERR_INVALID;
  }
  if (device < 0 || drl_device_count() <= device) { set_error("CUDA device %d not available (no CPU fallback)", device); return DRL_ERR_CUDA; }
  return DRL_OK;
}

int replay_core_init(ReplayCore* r, int device, int64_t capacity) {
  r->device = device;
  r->capacity = capacity;
  r->levels = replay_tree_levels(capacity);
  DRL_CUDA_CHECK(cudaSetDevice(device));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&r->ev_last, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventRecord(r->ev_last, r->stream));
  DRL_TRY(dev_alloc(r, &r->tree, 2 * (size_t)capacity - 1));
  return DRL_OK;
}

void replay_core_release(ReplayCore* r) {
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
  r->allocs.clear();
  if (r->ev_last) cudaEventDestroy(r->ev_last);
  if (r->stream) cudaStreamDestroy(r->stream);
  cudaGetLastError();
}

int replay_acquire(PinnedBlock& b, size_t bytes) {
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

int replay_ensure_sample(ReplayCore* r, int n) {
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

int replay_ensure_ingest(ReplayCore* r, size_t bytes) {
  DRL_TRY(replay_acquire(r->ingest, bytes));
  if (bytes <= r->ingest_bytes) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  if (r->d_ingest) cudaFree(r->d_ingest);
  r->d_ingest = nullptr;
  r->ingest_bytes = 0;
  DRL_CUDA_CHECK(cudaMalloc(&r->d_ingest, bytes));
  r->ingest_bytes = bytes;
  return DRL_OK;
}

int replay_begin(ReplayCore* r, cudaStream_t s) {
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(s, r->ev_last, 0));
  return DRL_OK;
}

int replay_end(ReplayCore* r, cudaStream_t s) {
  DRL_CUDA_CHECK(cudaEventRecord(r->ev_last, s));
  return DRL_OK;
}

int replay_launch_update(ReplayCore* r, cudaStream_t s, int n, const int64_t* tree_index, int64_t first,
                         const double* err64, const float* err32) {
  prof_mark(s, "replay_tree_update");
  DRL_CUDA_CHECK((launch_k(replay_tree_update_kernel, 1, 32 * r->levels, 0, s, r->tree, r->capacity, n, tree_index,
                           first, err64, err32)));
  return DRL_OK;
}

int replay_launch_sample(ReplayCore* r, cudaStream_t s, int n, const double* u01_dev, float* weight32) {
  r->beta = fmin(1.0, r->beta + kReplayBetaInc);
  prof_mark(s, "replay_sample");
  DRL_CUDA_CHECK((launch_k(replay_sample_kernel, 1, 256, 0, s, r->tree, r->capacity, n, u01_dev, (double)r->n_entries,
                           r->beta, r->d_tree_index, r->d_data_index, r->d_priority, r->d_is_weight, weight32)));
  r->last_n = n;
  return DRL_OK;
}

int replay_check_u01(const ReplayCore* r, int n, const double* u01) {
  for (int i = 0; i < n; ++i)
    if (!(u01[i] >= 0.0 && u01[i] <= 1.0)) { set_error("%s: u01[%d] = %g is not in [0, 1]", r->family, i, u01[i]); return DRL_ERR_INVALID; }
  return DRL_OK;
}

void replay_advance(ReplayCore* r, int n) {
  r->cursor = (r->cursor + n) % r->capacity;                 // SumTree.add (:351-359)
  r->n_entries = std::min<int64_t>(r->capacity, r->n_entries + n);
}

int replay_step(ReplayCore* r, AdamLearner* learner, int slot, const double* u01, float* weight32, const float* td_dev,
                const std::function<int(cudaStream_t)>& gather) {
  if (!u01) { set_error("%s step: null u01", r->family); return DRL_ERR_INVALID; }
  if (r->n_entries < 1) { set_error("%s step: the memory is empty", r->family); return DRL_ERR_STATE; }
  const int B = learner->B;
  DRL_TRY(replay_check_u01(r, B, u01));
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(replay_ensure_sample(r, B));
  if ((int)r->uniforms.size() <= slot) r->uniforms.resize(slot + 1);
  PinnedBlock& ub = r->uniforms[slot];
  DRL_TRY(replay_acquire(ub, (size_t)B * 8));
  memcpy(ub.h, u01, (size_t)B * 8);
  const cudaStream_t s = learner->compute;
  LearnerSlot& sl = learner->slots[slot];
  DRL_TRY(replay_begin(r, s));
  if (sl.has_data) DRL_CUDA_CHECK(cudaStreamWaitEvent(s, sl.staged, 0));   // an earlier drl_*_stage of the slot
  DRL_TRY(replay_launch_sample(r, s, B, reinterpret_cast<const double*>(ub.d), weight32));
  DRL_CUDA_CHECK(cudaEventRecord(ub.ev, s));
  DRL_TRY(gather(s));
  DRL_CUDA_CHECK(cudaEventRecord(sl.staged, s));
  sl.has_data = true;
  DRL_TRY(learner_run_step(learner, slot));
  // Memory.update of the sampled leaves with the step's |td|, before drl_*_wait returns
  DRL_TRY(replay_launch_update(r, s, B, r->d_tree_index, 0, nullptr, td_dev));
  DRL_CUDA_CHECK(cudaEventRecord(learner->ev_done[learner->last_row], s));
  return replay_end(r, s);
}

int replay_sample(ReplayCore* r, const char* family, int32_t n, const double* u01, int64_t* tree_index,
                  int64_t* data_index, double* priority, double* is_weight) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || !u01 || !tree_index || !data_index || !priority || !is_weight) { set_error("%s sample: bad argument", family); return DRL_ERR_INVALID; }
  if (r->n_entries < 1) { set_error("%s sample: the memory is empty", family); return DRL_ERR_STATE; }
  DRL_TRY(replay_check_u01(r, n, u01));
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(replay_ensure_sample(r, n));
  DRL_TRY(replay_acquire(r->args, (size_t)n * 8));
  memcpy(r->args.h, u01, (size_t)n * 8);
  const cudaStream_t s = r->stream;
  DRL_TRY(replay_begin(r, s));
  DRL_TRY(replay_launch_sample(r, s, n, reinterpret_cast<const double*>(r->args.d), nullptr));
  DRL_CUDA_CHECK(cudaEventRecord(r->args.ev, s));
  DRL_TRY(replay_end(r, s));
  DRL_TRY(replay_last_sample(r, family, tree_index, priority, is_weight));
  DRL_CUDA_CHECK(cudaMemcpy(data_index, r->d_data_index, (size_t)n * 8, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int replay_update(ReplayCore* r, const char* family, int32_t n, const int64_t* tree_index, const double* error) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (n < 1 || !tree_index || !error) { set_error("%s update: bad argument", family); return DRL_ERR_INVALID; }
  for (int i = 0; i < n; ++i)
    if (tree_index[i] < r->capacity - 1 || tree_index[i] >= 2 * r->capacity - 1) {
      set_error("%s update: %lld is not a leaf index", family, (long long)tree_index[i]);
      return DRL_ERR_INVALID;
    }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_TRY(replay_acquire(r->args, (size_t)n * 16));
  memcpy(r->args.h, tree_index, (size_t)n * 8);
  memcpy(r->args.h + (size_t)n * 8, error, (size_t)n * 8);
  const cudaStream_t s = r->stream;
  DRL_TRY(replay_begin(r, s));
  DRL_TRY(replay_launch_update(r, s, n, reinterpret_cast<const int64_t*>(r->args.d), 0,
                               reinterpret_cast<const double*>(r->args.d + (size_t)n * 8), nullptr));
  DRL_CUDA_CHECK(cudaEventRecord(r->args.ev, s));
  return replay_end(r, s);
}

int replay_last_sample(ReplayCore* r, const char* family, int64_t* tree_index, double* priority, double* is_weight) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (r->last_n < 1) { set_error("%s last_sample: nothing has been sampled", family); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  const size_t bytes = (size_t)r->last_n * 8;
  if (tree_index) DRL_CUDA_CHECK(cudaMemcpy(tree_index, r->d_tree_index, bytes, cudaMemcpyDeviceToHost));
  if (priority) DRL_CUDA_CHECK(cudaMemcpy(priority, r->d_priority, bytes, cudaMemcpyDeviceToHost));
  if (is_weight) DRL_CUDA_CHECK(cudaMemcpy(is_weight, r->d_is_weight, bytes, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int replay_total(ReplayCore* r, const char* family, double* total) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!total) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_CUDA_CHECK(cudaSetDevice(r->device));
  DRL_CUDA_CHECK(cudaEventSynchronize(r->ev_last));
  DRL_CUDA_CHECK(cudaMemcpy(total, r->tree, 8, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int replay_size(ReplayCore* r, const char* family, int64_t* n_entries) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!n_entries) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n_entries = r->n_entries;
  return DRL_OK;
}

int replay_beta(ReplayCore* r, const char* family, double* beta) {
  DRL_TRY(replay_check(r, family));
  std::lock_guard<std::recursive_mutex> lk(r->mu);
  if (!beta) { set_error("null argument"); return DRL_ERR_INVALID; }
  *beta = r->beta;
  return DRL_OK;
}

}  // namespace drl
