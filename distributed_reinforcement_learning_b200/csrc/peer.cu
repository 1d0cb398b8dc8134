// peer.cu -- the data-parallel exchange of the learner step as kernels over NVLink peer memory (one process per
// GPU, buffers shared with CUDA IPC) instead of a library all-reduce between two graphs:
//
//   backward (every rank: local gradient bucket [grads | 3 loss sums])
//   peer_reduce      barrier 0 in its prologue (every rank flags every peer, waits for every peer's flag: all
//                    buckets complete); rank r owns slice r of the bucket: reads that slice from EVERY rank's bucket
//                    over NVLink, sums in rank order, writes the sum into every rank's `reduced` buffer and its
//                    partial squared norms into every rank's partial table (reduce-scatter + all-gather in one pass,
//                    (W-1)/W of the bucket in each direction per rank); also lr / global_step like the single-GPU
//                    norm kernel; its last CTA signals barrier 1
//   rmsprop_apply    waits for barrier 1 in its prologue (all slices and partials delivered, all reads of the buckets
//                    finished), then the usual clip by the global norm + TF1 RMSProp on the local `reduced` buffer
//
// The kernel takes a float4 sub-range and an instance number, so the exchange can be issued in pieces.  Issuing the
// 97 % of the bucket that is complete ~100 us before the backward pass ends (everything but the conv weights) on a
// third stream was tried: inside the CUDA graph the conv weight-gradient kernels then queued BEHIND the exchange
// kernel (tools/timeline.py), so nothing was hidden, and the small second piece still paid two flag round trips
// (~25 us).  One instance after the backward pass is what runs.
//
// Every element is summed by exactly one rank in a fixed order, so all replicas get bit-identical gradients.  The
// whole step (forward, backward, exchange, update) is ONE CUDA graph per slot; nothing on the host sits between the
// backward pass and the update.  Flags only ever grow (epoch counters), so nothing needs resetting; two barriers per
// step order every reuse of bucket / reduced / partials (see DESIGN.md section 5).
#include "kernels.h"
#include "peer_sync.cuh"

namespace drl { constexpr int kPeerThreads = 256; }

namespace drl {

// Barrier 0 + reduce-scatter + all-gather + partial norms + the signal of barrier 1, one launch:
//   prologue  CTA 0 tells every peer "my bucket is complete" (it is: the backward pass precedes this kernel on the
//             stream); every CTA waits until all peers have said so
//   body      slice `rank` of the range, 8 independent float4 per thread in flight per peer (a remote load takes
//             ~3 us; tools/microbench/p2p_bw.cu: 8 MB over NVLink costs ~22 us per direction, launch included)
//   epilogue  the last CTA to finish (ticket counter, fence before the ticket) publishes the epochs and tells every
//             peer "my slice and my partials have been delivered to you"; the update kernel waits for those flags.
__global__ void __launch_bounds__(kPeerThreads) peer_reduce_kernel(PeerTable t, OptState o, int rank, int world, int nblk_r,
                                                          int part, int64_t beg4, int64_t end4, int do_lr) {
  kernel_prologue();
  __shared__ float red[8];
  __shared__ bool last_s;
  uint32_t* epoch = t.epoch[rank] + 4 * part; // [0], [1]: epochs completed; [2]: ticket counter
  const uint32_t e = epoch[0] + 1;            // stable while this kernel runs: only its last CTA writes it
  const int ph_ready = 2 * part, ph_done = 2 * part + 1;
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(t.flags[threadIdx.x] + ph_ready * kMaxPeers + rank, e);
  }
  const PeerErr perr{t.err[rank], t.err_host, t.timeout_ns};
  // failed state (now or earlier): leave every buffer, the step counter and the epochs untouched (see peer_sync.cuh)
  if (!wait_peers(t.flags[rank], ph_ready, world, e, perr)) return;

  const int64_t n4_grad = o.n / 4;            // gradients (the norm is over these; the bucket tail holds loss sums)
  const int64_t per = (end4 - beg4 + world - 1) / world;
  const int64_t beg = beg4 + per * rank, end = min(end4, beg + per);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  float acc = 0.f;
  constexpr int U = 8;
  for (int64_t i0 = beg + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < end; i0 += U * stride) {
    float4 s[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      s[u] = (i < end) ? __ldcg(reinterpret_cast<const float4*>(t.bucket[0]) + i) : zero4();
    }
    for (int p = 1; p < world; ++p) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = (i < end) ? __ldcg(reinterpret_cast<const float4*>(t.bucket[p]) + i) : zero4();
      }
#pragma unroll
      for (int u = 0; u < U; ++u) { s[u].x += v[u].x; s[u].y += v[u].y; s[u].z += v[u].z; s[u].w += v[u].w; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < end) {
        for (int p = 0; p < world; ++p) reinterpret_cast<float4*>(t.reduced[p])[i] = s[u];
        if (i < n4_grad) {
          acc = fmaf(s[u].x, s[u].x, acc); acc = fmaf(s[u].y, s[u].y, acc);
          acc = fmaf(s[u].z, s[u].z, acc); acc = fmaf(s[u].w, s[u].w, acc);
        }
      }
    }
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kPeerThreads / 32; ++i) s += red[i];
    for (int p = 0; p < world; ++p) t.partials[p][(part * world + rank) * nblk_r + blockIdx.x] = s;
    if (blockIdx.x == 0 && do_lr) {      // tf.train.polynomial_decay in float32 (agent/impala.py:96), pre-increment step
      const long long step = *o.step;
      const float decay = (float)o.learning_frame;
      const float gs = fminf((float)step, decay);
      const float pp = gs / decay;
      *o.lr_cur = (o.start_lr - o.end_lr) * (1.0f - pp) + o.end_lr;
      *o.step = step + 1;
    }
  }
  // ---- last CTA: everything this rank had to deliver has been written -> barrier-1 signal ----
  __threadfence_system();                                     // every thread: its remote stores before the CTA's ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    const uint32_t ticket = atomicAdd(&epoch[2], 1u);
    last_s = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (last_s) {
    if (threadIdx.x == 0) { epoch[0] = e; epoch[1] = e; epoch[2] = 0u; }
    if (threadIdx.x < world) {
      __threadfence_system();
      st_release_sys(t.flags[threadIdx.x] + ph_done * kMaxPeers + rank, e);
    }
  }
}

// one exchange instance; the update kernel waits for every instance's "delivered" flags in its prologue
int peer_exchange(cudaStream_t s, const PeerPlan& pp, int part, int64_t beg4, int64_t end4, bool do_lr, int grid) {
  // grid <= pp.nblk: the partial-norm table has pp.nblk entries per (part, rank); a smaller grid leaves the rest at their
  // initial zeros (the grid of a part never changes during the handle's life)
  if (grid <= 0 || grid > pp.nblk) grid = pp.nblk;
  DRL_CUDA_CHECK((launch_k(peer_reduce_kernel, grid, kPeerThreads, 0, s, pp.t, pp.o, pp.rank, pp.world, pp.nblk, part, beg4, end4,
                           do_lr ? 1 : 0)));
  return DRL_OK;
}

}  // namespace drl
