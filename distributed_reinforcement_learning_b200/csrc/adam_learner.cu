// adam_learner.cu -- TF1 Adam and the learner-handle core of the Ape-X / A3C and the R2D2 handles (adam_learner.cuh).
#include <string.h>

#include "adam_learner.cuh"
#include "gemm_umma.cuh"
#include "loaders.cuh"
#include "trunk_images.cuh"

namespace drl {

// ------------------------------------------------------------------------------------------
// Tail of the train op (agent/apex.py:70-75) with TF 1.14 semantics:
//   lr    = polynomial_decay(start, global_step, decay_steps, end)      (float32, pre-increment step)
//   g    <- g * clip * min(1/||g||, 1/clip)                              (clip_by_global_norm over the main variables;
//                                                                         the target variables have gradient None)
//   alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)               (ApplyAdam, float32)
//   m    += (g - m)(1 - beta1) ; v += (g^2 - v)(1 - beta2) ; w -= m * alpha / (sqrt(v) + eps)
//   beta powers *= beta ; global_step += 1
// Two launches: (1) partial squared norms + the scalars, (2) every block re-reduces the partials in fixed order.
// ------------------------------------------------------------------------------------------
constexpr float kBeta1 = 0.9f, kBeta2 = 0.999f, kAdamEps = 1e-8f;

__global__ void __launch_bounds__(256) adam_prepare_kernel(AdamState o) {
  kernel_prologue();
  __shared__ float red[8];
  const int64_t n4 = o.n / 4;
  const float4* g4 = reinterpret_cast<const float4*>(o.grads);
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = g4[i];
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc); acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i];
    o.norm_partials[blockIdx.x] = s;
    if (blockIdx.x == 0) {
      const long long step = *o.step;
      const float decay = (float)o.learning_frame;
      const float gs = fminf((float)step, decay);
      const float p = gs / decay;
      const float lr = (o.start_lr - o.end_lr) * (1.0f - p) + o.end_lr;
      const float b1 = *o.b1p, b2 = *o.b2p;
      *o.lr_cur = lr;
      *o.alpha = lr * sqrtf(1.0f - b2) / (1.0f - b1);
      *o.b1p = b1 * kBeta1;
      *o.b2p = b2 * kBeta2;
      *o.step = step + 1;
    }
  }
}

__global__ void __launch_bounds__(256) adam_apply_kernel(AdamState o) {
  kernel_prologue();
  __shared__ float red[8];
  __shared__ float s_scale;
  float acc = 0.f;
  for (int i = threadIdx.x; i < o.nblk; i += blockDim.x) acc += o.norm_partials[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i];
    const float norm = sqrtf(s) * o.grad_scale;
    s_scale = ((o.clip_norm > 0.f) ? o.clip_norm * fminf(1.0f / norm, 1.0f / o.clip_norm) : 1.0f) * o.grad_scale;
    if (blockIdx.x == 0) {
      o.out[0] = o.loss[0] * o.grad_scale; o.out[1] = *o.lr_cur; o.out[2] = norm;
      o.out[3] = o.loss[1] * o.grad_scale; o.out[4] = o.loss[2] * o.grad_scale;          // A3C: baseline loss, entropy (zero for the DQN learners)
      const long long st = *o.step;
      o.out[6] = __int_as_float((int)(st & 0xffffffffll));
      o.out[7] = __int_as_float((int)(st >> 32));
    }
  }
  __syncthreads();
  const float scale = s_scale;
  const float alpha = *o.alpha;
  const int64_t n4 = o.n / 4;
  const float4* g4 = reinterpret_cast<const float4*>(o.grads);
  float4* w4 = reinterpret_cast<float4*>(o.params);
  float4* m4 = reinterpret_cast<float4*>(o.m);
  float4* v4 = reinterpret_cast<float4*>(o.v);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 g = g4[i];
    float4 m = m4[i], v = v4[i], w = w4[i];
    float gg;
    gg = g.x * scale; m.x += (gg - m.x) * (1.0f - kBeta1); v.x += (gg * gg - v.x) * (1.0f - kBeta2); w.x -= (m.x * alpha) / (sqrtf(v.x) + kAdamEps);
    gg = g.y * scale; m.y += (gg - m.y) * (1.0f - kBeta1); v.y += (gg * gg - v.y) * (1.0f - kBeta2); w.y -= (m.y * alpha) / (sqrtf(v.y) + kAdamEps);
    gg = g.z * scale; m.z += (gg - m.z) * (1.0f - kBeta1); v.z += (gg * gg - v.z) * (1.0f - kBeta2); w.z -= (m.z * alpha) / (sqrtf(v.z) + kAdamEps);
    gg = g.w * scale; m.w += (gg - m.w) * (1.0f - kBeta1); v.w += (gg * gg - v.w) * (1.0f - kBeta2); w.w -= (m.w * alpha) / (sqrtf(v.w) + kAdamEps);
    m4[i] = m; v4[i] = v; w4[i] = w;
  }
}

int adam_step(cudaStream_t s, const AdamState& o) {
  DRL_CUDA_CHECK((launch_k(adam_prepare_kernel, o.nblk, 256, 0, s, o)));
  DRL_CUDA_CHECK((launch_k(adam_apply_kernel, o.nblk, 256, 0, s, o)));
  return DRL_OK;
}

// ---- handle core ----------------------------------------------------------------------------

Streams AdamLearner::streams() const {
  Streams st;
  st.main = compute;
  st.side = side;
  for (int i = 0; i < 8; ++i) st.ev[i] = fj[i];
  st.par = par;
  return st;
}

Streams AdamLearner::target_streams() const {
  Streams st;
  st.main = par ? tmain : compute;
  st.side = par ? tside : side;
  for (int i = 0; i < 8; ++i) st.ev[i] = par ? tfj[i] : fj[i];
  st.par = par;
  return st;
}

int adam_learner_init(AdamLearner* h, size_t slot_bytes, size_t ones) {
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->compute, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->copy, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
  for (int i = 0; i < 8; ++i) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->fj[i], cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->tmain, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->tside, cudaStreamNonBlocking));
  for (int i = 0; i < 8; ++i) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->tfj[i], cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_tfork, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_tjoin, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreate(&h->ev_start));
  DRL_CUDA_CHECK(cudaEventCreate(&h->ev_stop));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_done, cudaEventDisableTiming));
  const size_t B = h->B, NP = h->layout->padded_total;
  DRL_TRY(dev_alloc(h, &h->params, NP));
  DRL_TRY(dev_alloc(h, &h->target, NP));
  DRL_TRY(dev_alloc(h, &h->adam_m, NP));
  DRL_TRY(dev_alloc(h, &h->adam_v, NP));
  DRL_TRY(dev_alloc(h, &h->grads, NP + 4));
  h->loss = h->grads + NP;
  {
    size_t wb[WeightImages::kCount];
    weight_image_sizes(wb);
    for (int i : {1, 2, 5, 6}) DRL_TRY(dev_alloc(h, &h->wi.img[i], wb[i]));
    for (int i : {1, 2}) DRL_TRY(dev_alloc(h, &h->twi.img[i], wb[i]));
  }
  DRL_TRY(dev_alloc(h, &h->d_step, 1));
  DRL_TRY(dev_alloc(h, &h->d_lr, 1));
  DRL_TRY(dev_alloc(h, &h->d_alpha, 1));
  DRL_TRY(dev_alloc(h, &h->d_b1p, 1));
  DRL_TRY(dev_alloc(h, &h->d_b2p, 1));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b1p, &kBeta1, 4, cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b2p, &kBeta2, 4, cudaMemcpyHostToDevice));
  const size_t ns = h->num_slots;
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_out, ns * 8 * sizeof(float), cudaHostAllocMapped));
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_out, h->h_out, 0));
  memset(h->h_out, 0, ns * 8 * sizeof(float));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_td, ns * B * sizeof(float), cudaHostAllocMapped));
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_td, h->h_td, 0));
  memset(h->h_td, 0, ns * B * sizeof(float));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_flat, NP * sizeof(float), cudaHostAllocDefault));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_ones, ones * sizeof(float), cudaHostAllocDefault));
  for (size_t i = 0; i < ones; ++i) h->h_ones[i] = 1.0f;
  AdamState& o = h->opt;
  o.params = h->params; o.m = h->adam_m; o.v = h->adam_v; o.grads = h->grads; o.n = (int64_t)NP;
  o.nblk = 132 * 4;
  DRL_TRY(dev_alloc(h, &o.norm_partials, o.nblk));
  o.step = h->d_step; o.lr_cur = h->d_lr; o.alpha = h->d_alpha; o.b1p = h->d_b1p; o.b2p = h->d_b2p;
  o.out = h->d_out; o.loss = h->loss;
  o.grad_scale = 1.0f;
  h->slots.resize(ns + 1);
  h->graph_step.assign(ns, nullptr);
  for (AdamSlot& s : h->slots) {
    DRL_TRY(dev_alloc(h, &s.base, slot_bytes));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&s.staged, cudaEventDisableTiming));
    DRL_CUDA_CHECK(cudaEventCreateWithFlags(&s.consumed, cudaEventDisableTiming));
  }
  return DRL_OK;
}

void adam_learner_release(AdamLearner* h) {
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (auto g : h->graph_step) if (g) cudaGraphExecDestroy(g);
  for (AdamSlot& s : h->slots) {
    if (s.staged) cudaEventDestroy(s.staged);
    if (s.consumed) cudaEventDestroy(s.consumed);
  }
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_out) cudaFreeHost(h->h_out);
  if (h->h_td) cudaFreeHost(h->h_td);
  if (h->h_flat) cudaFreeHost(h->h_flat);
  if (h->h_ones) cudaFreeHost(h->h_ones);
  if (h->ev_start) cudaEventDestroy(h->ev_start);
  if (h->ev_stop) cudaEventDestroy(h->ev_stop);
  if (h->ev_done) cudaEventDestroy(h->ev_done);
  for (int i = 0; i < 8; ++i) if (h->fj[i]) cudaEventDestroy(h->fj[i]);
  for (int i = 0; i < 8; ++i) if (h->tfj[i]) cudaEventDestroy(h->tfj[i]);
  if (h->ev_tfork) cudaEventDestroy(h->ev_tfork);
  if (h->ev_tjoin) cudaEventDestroy(h->ev_tjoin);
  if (h->tmain) cudaStreamDestroy(h->tmain);
  if (h->tside) cudaStreamDestroy(h->tside);
  if (h->side) cudaStreamDestroy(h->side);
  if (h->compute) cudaStreamDestroy(h->compute);
  if (h->copy) cudaStreamDestroy(h->copy);
  cudaGetLastError();
}

namespace {

int set_device(const AdamLearner* h) {
  DRL_CUDA_CHECK(cudaSetDevice(h->device));
  return DRL_OK;
}

int upload(AdamLearner* h, float* dev_padded, const float* host_packed) {
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  return upload_flat(h->compute, h->h_flat, *h->layout, dev_padded, host_packed, 0.0f);
}
int download(AdamLearner* h, const float* dev_padded, float* host_packed) {
  return download_flat(h->compute, h->h_flat, *h->layout, dev_padded, host_packed);
}

int check_which(int which) {
  if (which != 0 && which != 1) { set_error("which must be 0 (main) or 1 (target)"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

// the main images follow the parameters, which change every step; the target images only change with the target
// copy / set_params.  Refreshed outside of the graph so that the captured step never contains them.
int refresh_target_images(AdamLearner* h) {
  if (h->target_images_stale && h->mode >= 2) {
    DRL_TRY(conv_images_tf32(h->compute, *h->layout, h->target, h->twi.img[1], h->twi.img[2]));
  }
  h->target_images_stale = false;
  return DRL_OK;
}

int enqueue_step(AdamLearner* h, int slot, int* launches) {
  DRL_TRY(h->fwd_bwd(h, slot, launches));
  AdamState o = h->opt;
  o.out = h->d_out + 8 * slot;
  prof_mark(h->compute, "optimizer(norm+adam)");
  DRL_TRY(adam_step(h->compute, o));
  prof_mark(h->compute, "end");
  if (launches) *launches += 2;
  return DRL_OK;
}

int wait_staged(AdamLearner* h, int slot) {
  const AdamSlot& sl = h->slots[slot];
  if (!sl.has_data) { set_error("slot %d has not been staged", slot); return DRL_ERR_STATE; }
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, sl.staged, 0));
  return DRL_OK;
}

}  // namespace

int adam_run_step(AdamLearner* h, int slot) {
  DRL_TRY(wait_staged(h, slot));
  if (h->use_cuda_graph) DRL_TRY(refresh_target_images(h));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->compute));
  h->main_images_stale = true;
  int cnt = 0;
  if (h->use_cuda_graph) {
    if (!h->graph_step[slot]) {
      // eager pass of forward + loss + backward first (sets the per-kernel attributes outside of capture; it does not
      // change any state the captured pass depends on: parameters and optimizer state are only touched by the update)
      DRL_TRY(h->fwd_bwd(h, slot, nullptr));
      h->main_images_stale = true;
      DRL_TRY(capture_graph(h->compute, [&] { return enqueue_step(h, slot, &cnt); }, &h->graph_step[slot]));
      h->launches = cnt;
    }
    DRL_CUDA_CHECK(cudaGraphLaunch(h->graph_step[slot], h->compute));
  } else {
    DRL_TRY(enqueue_step(h, slot, &cnt));
    h->launches = cnt;
  }
  h->main_images_stale = true;      // the update changed the main parameters
  h->last_n = h->B;
  h->last_slot = slot;
  DRL_CUDA_CHECK(cudaEventRecord(h->slots[slot].consumed, h->compute));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->compute));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_done, h->compute));
  h->pending = true;
  return DRL_OK;
}

int check_handle(const AdamLearner* h, const char* family) {
  if (!h) { set_error("null %s handle", family); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int check_slot(const AdamLearner* h, int slot) {
  if (slot < 0 || slot >= h->num_slots) { set_error("slot %d out of range", slot); return DRL_ERR_INVALID; }
  return DRL_OK;
}

int64_t step_of(const float* row) {
  uint32_t lo, hi;
  memcpy(&lo, &row[6], 4);
  memcpy(&hi, &row[7], 4);
  return (int64_t)(((uint64_t)hi << 32) | lo);
}

int adam_param_count(const AdamLearner* h, const char* family, int64_t* n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->layout->packed_total;
  return DRL_OK;
}

int adam_set_params(AdamLearner* h, const char* family, int which, const float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_which(which));
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("set_params: expected %lld floats, got %lld", (long long)np, (long long)n); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(upload(h, which == 0 ? h->params : h->target, host_flat));
  if (which == 0) h->main_images_stale = true; else h->target_images_stale = true;
  return DRL_OK;
}

int adam_get_params(AdamLearner* h, const char* family, int which, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_which(which));
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("get_params: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  return download(h, which == 0 ? h->params : h->target, host_flat);
}

int adam_set_opt_state(AdamLearner* h, const char* family, const float* host_m, const float* host_v, int64_t n,
                       int64_t step, float beta1_power, float beta2_power) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_m || !host_v || n != np) { set_error("set_opt_state: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(upload(h, h->adam_m, host_m));
  DRL_TRY(upload(h, h->adam_v, host_v));
  long long st = step;
  DRL_CUDA_CHECK(cudaMemcpy(h->d_step, &st, sizeof(st), cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b1p, &beta1_power, 4, cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b2p, &beta2_power, 4, cudaMemcpyHostToDevice));
  return DRL_OK;
}

int adam_get_opt_state(AdamLearner* h, const char* family, float* host_m, float* host_v, int64_t n, int64_t* step,
                       float* beta1_power, float* beta2_power) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (n != np) { set_error("get_opt_state: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  if (host_m) DRL_TRY(download(h, h->adam_m, host_m));
  if (host_v) DRL_TRY(download(h, h->adam_v, host_v));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  if (step) {
    long long st = 0;
    DRL_CUDA_CHECK(cudaMemcpy(&st, h->d_step, sizeof(st), cudaMemcpyDeviceToHost));
    *step = st;
  }
  if (beta1_power) DRL_CUDA_CHECK(cudaMemcpy(beta1_power, h->d_b1p, 4, cudaMemcpyDeviceToHost));
  if (beta2_power) DRL_CUDA_CHECK(cudaMemcpy(beta2_power, h->d_b2p, 4, cudaMemcpyDeviceToHost));
  return DRL_OK;
}

int adam_get_grads(AdamLearner* h, const char* family, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("get_grads: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  return download(h, h->grads, host_flat);
}

int adam_main_to_target(AdamLearner* h, const char* family) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->target, h->params, h->layout->padded_total * sizeof(float), cudaMemcpyDeviceToDevice,
                                 h->compute));
  h->target_images_stale = true;
  return DRL_OK;
}

int adam_params_snapshot(AdamLearner* h, const char* family, int device, cudaStream_t dst_stream, float* dst,
                         cudaEvent_t ev_ready, cudaEvent_t ev_copied) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (h->device != device) {
    set_error("sync: the learner is on device %d, the policy on device %d (no cross-device sync)", h->device, device);
    return DRL_ERR_INVALID;
  }
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaEventRecord(ev_ready, h->compute));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(dst_stream, ev_ready, 0));
  DRL_CUDA_CHECK(cudaMemcpyAsync(dst, h->params, (size_t)h->layout->padded_total * sizeof(float),
                                 cudaMemcpyDeviceToDevice, dst_stream));
  DRL_CUDA_CHECK(cudaEventRecord(ev_copied, dst_stream));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(h->compute, ev_copied, 0));
  return DRL_OK;
}

int adam_step_async(AdamLearner* h, const char* family, int slot) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  return adam_run_step(h, slot);
}

// data parallel: the step in two halves around the caller's all-reduce of the bucket (eager launches)
int adam_forward_backward(AdamLearner* h, const char* family, int slot) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  DRL_TRY(set_device(h));
  DRL_TRY(wait_staged(h, slot));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_start, h->compute));
  h->main_images_stale = true;
  int cnt = 0;
  DRL_TRY(h->fwd_bwd(h, slot, &cnt));
  h->launches = cnt + 2;
  h->last_n = h->B;
  h->last_slot = slot;
  DRL_CUDA_CHECK(cudaEventRecord(h->slots[slot].consumed, h->compute));
  return DRL_OK;
}

int adam_grad_bucket(AdamLearner* h, const char* family, void** dev_ptr, int64_t* count) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (dev_ptr) *dev_ptr = h->grads;
  if (count) *count = h->layout->padded_total + 4;
  return DRL_OK;
}

int adam_apply(AdamLearner* h, const char* family, float grad_scale) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!(grad_scale > 0.f)) { set_error("apply: grad_scale must be > 0"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  AdamState o = h->opt;
  o.out = h->d_out + 8 * h->last_slot;
  o.grad_scale = grad_scale;
  DRL_TRY(adam_step(h->compute, o));
  h->main_images_stale = true;
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_stop, h->compute));
  DRL_CUDA_CHECK(cudaEventRecord(h->ev_done, h->compute));
  h->pending = true;
  return DRL_OK;
}

int adam_wait(AdamLearner* h, const char* family, const float** row, float* td_error) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!h->pending) { set_error("wait: no step in flight"); return DRL_ERR_STATE; }
  DRL_TRY(set_device(h));
  h->pending = false;
  DRL_CUDA_CHECK(cudaEventSynchronize(h->ev_done));
  *row = h->h_out + 8 * h->last_slot;
  if (td_error) memcpy(td_error, h->h_td + (size_t)h->last_slot * h->B, (size_t)h->B * sizeof(float));
  return DRL_OK;
}

int adam_profile_step(AdamLearner* h, const char* family, int slot, char* names, int64_t names_len, float* ms,
                      int32_t max_kernels, int32_t* count) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_slot(h, slot));
  if (!names || !ms || !count) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(wait_staged(h, slot));
  DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
  prof_begin();
  const bool par_saved = h->par;
  h->par = false;
  h->main_images_stale = true;
  int rc = enqueue_step(h, slot, nullptr);
  h->par = par_saved;
  h->main_images_stale = true;
  h->last_n = h->B;
  DRL_TRY(prof_end(h->compute, rc, names, names_len, ms, max_kernels, count));
  h->pending = false;
  return DRL_OK;
}

int adam_last_step_ms(AdamLearner* h, const char* family, float* ms) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!ms) { set_error("null argument"); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaEventSynchronize(h->ev_stop));
  DRL_CUDA_CHECK(cudaEventElapsedTime(ms, h->ev_start, h->ev_stop));
  return DRL_OK;
}

int adam_stream(AdamLearner* h, const char* family, void** stream) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!stream) { set_error("null argument"); return DRL_ERR_INVALID; }
  *stream = h->compute;
  return DRL_OK;
}

int adam_launches_per_step(const AdamLearner* h, const char* family, int32_t* n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  if (!n) { set_error("null argument"); return DRL_ERR_INVALID; }
  *n = h->launches;     // valid after the first step
  return DRL_OK;
}

int read_named_buffer(AdamLearner* h, const NamedBuffer* tab, int ntab, const char* name, float* host_dst, int64_t n) {
  for (int i = 0; i < ntab; ++i) {
    const NamedBuffer& e = tab[i];
    if (strcmp(e.name, name) != 0) continue;
    if ((size_t)n != e.count) { set_error("read_buffer(%s): expected %zu floats, got %lld", name, e.count, (long long)n); return DRL_ERR_INVALID; }
    DRL_CUDA_CHECK(cudaStreamSynchronize(h->compute));
    DRL_CUDA_CHECK(cudaMemcpy(host_dst, e.p, e.count * sizeof(float), cudaMemcpyDeviceToHost));
    return DRL_OK;
  }
  set_error("read_buffer: unknown buffer '%s'", name);
  return DRL_ERR_INVALID;
}

}  // namespace drl
