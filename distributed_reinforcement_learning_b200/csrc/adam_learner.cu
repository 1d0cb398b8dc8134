// adam_learner.cu -- TF1 Adam and the Adam layer of the Ape-X / A3C and the R2D2 handles (adam_learner.cuh).
#include <string.h>

#include "adam_learner.cuh"
#include "gemm_umma.cuh"
#include "loaders.cuh"
#include "trunk_images.cuh"

namespace drl {

// ------------------------------------------------------------------------------------------
// Tail of the train op (agent/apex.py:70-75) with TF 1.14 semantics:
//   lr    = polynomial_decay(start, global_step, decay_steps, end)      (float32, pre-increment step)
//   g    <- g * (clip * min(1/||g||, 1/clip) + (||g|| - ||g||))          (clip_by_global_norm over the main variables;
//                                                                         the target variables have gradient None; a NaN
//                                                                         or infinite norm makes every gradient NaN)
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
      const float lr = __fmul_rn(o.start_lr - o.end_lr, 1.0f - p) + o.end_lr;   // TF rounds the product: no FMA
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
    s_scale = ((o.clip_norm > 0.f) ? o.clip_norm * fminf(1.0f / norm, 1.0f / o.clip_norm) + (norm - norm) : 1.0f) *
              o.grad_scale;
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


// ---- Adam layer -----------------------------------------------------------------------------

Streams AdamLearner::target_streams() const {
  Streams st;
  st.main = par ? tmain : compute;
  st.side = par ? tside : side;
  for (int i = 0; i < 8; ++i) st.ev[i] = par ? tfj[i] : fj[i];
  st.par = par;
  return st;
}

namespace {

int update(LearnerCore* core, int out_row, float grad_scale, bool, bool) {
  AdamLearner* h = static_cast<AdamLearner*>(core);
  AdamState o = h->opt;
  o.out = h->d_out + 8 * out_row;
  o.grad_scale = grad_scale;
  prof_mark(h->compute, "optimizer(norm+adam)");
  DRL_TRY(adam_step(h->compute, o));
  prof_mark(h->compute, "end");
  return DRL_OK;
}

}  // namespace

int adam_learner_init(AdamLearner* h, size_t slot_bytes, size_t ones) {
  h->scratch_slots = 1;
  h->update = update;
  DRL_TRY(learner_core_init(h, slot_bytes));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->tmain, cudaStreamNonBlocking));
  DRL_CUDA_CHECK(cudaStreamCreateWithFlags(&h->tside, cudaStreamNonBlocking));
  for (int i = 0; i < 8; ++i) DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->tfj[i], cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_tfork, cudaEventDisableTiming));
  DRL_CUDA_CHECK(cudaEventCreateWithFlags(&h->ev_tjoin, cudaEventDisableTiming));
  const size_t B = h->B, NP = h->layout->padded_total;
  DRL_TRY(dev_alloc(h, &h->target, NP));
  DRL_TRY(dev_alloc(h, &h->adam_m, NP));
  DRL_TRY(dev_alloc(h, &h->adam_v, NP));
  {
    size_t wb[WeightImages::kCount];
    weight_image_sizes(wb);
    for (int i : {1, 2, 5, 6}) DRL_TRY(dev_alloc(h, &h->wi.img[i], wb[i]));
    for (int i : {1, 2}) DRL_TRY(dev_alloc(h, &h->twi.img[i], wb[i]));
  }
  DRL_TRY(dev_alloc(h, &h->d_alpha, 1));
  DRL_TRY(dev_alloc(h, &h->d_b1p, 1));
  DRL_TRY(dev_alloc(h, &h->d_b2p, 1));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b1p, &kBeta1, 4, cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemcpy(h->d_b2p, &kBeta2, 4, cudaMemcpyHostToDevice));
  const size_t ns = h->num_slots;
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_td, ns * B * sizeof(float), cudaHostAllocMapped));
  DRL_CUDA_CHECK(cudaHostGetDevicePointer((void**)&h->d_td, h->h_td, 0));
  memset(h->h_td, 0, ns * B * sizeof(float));
  DRL_CUDA_CHECK(cudaHostAlloc((void**)&h->h_ones, ones * sizeof(float), cudaHostAllocDefault));
  for (size_t i = 0; i < ones; ++i) h->h_ones[i] = 1.0f;
  AdamState& o = h->opt;
  o.params = h->params; o.m = h->adam_m; o.v = h->adam_v; o.grads = h->grads; o.n = (int64_t)NP;
  o.nblk = 132 * 4;
  DRL_TRY(dev_alloc(h, &o.norm_partials, o.nblk));
  o.step = h->d_step; o.lr_cur = h->d_lr; o.alpha = h->d_alpha; o.b1p = h->d_b1p; o.b2p = h->d_b2p;
  o.out = h->d_out; o.loss = h->loss;
  o.grad_scale = 1.0f;
  return DRL_OK;
}

void adam_learner_release(AdamLearner* h) {
  learner_core_release(h);
  if (h->h_td) cudaFreeHost(h->h_td);
  if (h->h_ones) cudaFreeHost(h->h_ones);
  for (int i = 0; i < 8; ++i) if (h->tfj[i]) cudaEventDestroy(h->tfj[i]);
  if (h->ev_tfork) cudaEventDestroy(h->ev_tfork);
  if (h->ev_tjoin) cudaEventDestroy(h->ev_tjoin);
  if (h->tmain) cudaStreamDestroy(h->tmain);
  if (h->tside) cudaStreamDestroy(h->tside);
  cudaGetLastError();
}

namespace {

int check_which(int which) {
  if (which != 0 && which != 1) { set_error("which must be 0 (main) or 1 (target)"); return DRL_ERR_INVALID; }
  return DRL_OK;
}

// The main images follow the parameters, which change every step; the target images only change with the target
// copy / set_params.  An eager forward rebuilds stale target images itself.  A captured step never contains that
// rebuild (the first step's eager pass, which runs before the capture, does it), so under use_cuda_graph the images are
// rebuilt here, outside of any graph, as soon as the target parameters change.
int target_changed(AdamLearner* h) {
  h->target_images_stale = true;
  if (!h->use_cuda_graph) return DRL_OK;
  if (h->mode >= 2) DRL_TRY(conv_images_tf32(h->compute, *h->layout, h->target, h->twi.img[1], h->twi.img[2]));
  h->target_images_stale = false;
  return DRL_OK;
}

}  // namespace

int adam_set_params(AdamLearner* h, const char* family, int which, const float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_which(which));
  if (which == 0) return learner_set_params(h, family, host_flat, n);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("set_params: expected %lld floats, got %lld", (long long)np, (long long)n); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(learner_upload(h, h->target, host_flat, 0.0f));
  return target_changed(h);
}

int adam_get_params(AdamLearner* h, const char* family, int which, float* host_flat, int64_t n) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(check_which(which));
  if (which == 0) return learner_get_params(h, family, host_flat, n);
  const int64_t np = h->layout->packed_total;
  if (!host_flat || n != np) { set_error("get_params: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  return learner_download(h, h->target, host_flat);
}

int adam_set_opt_state(AdamLearner* h, const char* family, const float* host_m, const float* host_v, int64_t n,
                       int64_t step, float beta1_power, float beta2_power) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  const int64_t np = h->layout->packed_total;
  if (!host_m || !host_v || n != np) { set_error("set_opt_state: expected %lld floats", (long long)np); return DRL_ERR_INVALID; }
  DRL_TRY(set_device(h));
  DRL_TRY(learner_upload(h, h->adam_m, host_m, 0.0f));
  DRL_TRY(learner_upload(h, h->adam_v, host_v, 0.0f));
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
  if (host_m) DRL_TRY(learner_download(h, h->adam_m, host_m));
  if (host_v) DRL_TRY(learner_download(h, h->adam_v, host_v));
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

int adam_main_to_target(AdamLearner* h, const char* family) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(set_device(h));
  DRL_CUDA_CHECK(cudaMemcpyAsync(h->target, h->params, h->layout->padded_total * sizeof(float), cudaMemcpyDeviceToDevice,
                                 h->compute));
  return target_changed(h);
}

int adam_wait(AdamLearner* h, const char* family, const float** row, float* td_error) {
  DRL_TRY(check_handle(h, family));
  std::lock_guard<std::recursive_mutex> lk(h->mu);
  DRL_TRY(learner_wait(h, family, row));
  if (td_error) memcpy(td_error, h->h_td + (size_t)h->last_slot * h->B, (size_t)h->B * sizeof(float));
  return DRL_OK;
}

}  // namespace drl
