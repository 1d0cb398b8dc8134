// replay_tree.cuh -- device sum tree of a prioritized replay memory (DESIGN.md section 10), independent of what the
// transitions are: the float64 tree of buffer_queue.SumTree (distributed_queue/buffer_queue.py:326-371), 2 * capacity - 1
// nodes with the leaves at [capacity - 1, 2 * capacity - 1), and the two kernels that read and write it, with the
// arithmetic of the host tree (per.cu) and the reference's Memory (:371-415).  The host keeps n_entries, the write
// cursor and beta, which follow from the call sequence alone, and passes them in; only the tree lives on the device.
#pragma once
#include "common.cuh"

namespace drl {

constexpr double kReplayE = 0.001, kReplayA = 0.6, kReplayBetaInc = 0.001;   // Memory.e / a / beta increment (:373-376)
// One warp per tree level in the update kernel: depth(2 * capacity - 2) <= 32 levels below the root.
constexpr int64_t kReplayMaxCapacity = int64_t(1) << 31;

// depth of node x (root 0): floor(log2(x + 1))
__device__ __forceinline__ int tree_depth(int64_t x) { return 63 - __clzll((unsigned long long)(x + 1)); }

// number of levels above the deepest leaf = depth(2 * capacity - 2): the warps of replay_tree_update_kernel
inline int replay_tree_levels(int64_t capacity) {
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

}  // namespace drl
