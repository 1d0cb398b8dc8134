// elementwise.cu -- the small kernels around the contractions: action-embedding table,
// LSTM gate nonlinearity (TF1 LSTMCell: gate order i,j,f,o, forget_bias 1.0), output heads
// (logits/softmax/value), their backward counterparts, and the split-K reduction.
#include <algorithm>

#include "kernels.h"

namespace drl {

// ------------------------------------------------------------------------------------------
// action_embedding (model/impala_actor_critic.py:12-16) evaluated once per distinct action:
//   e1[a]    = relu(W1[a,:] + b1)            (one_hot(a) @ W1 is row a of W1)
//   table[a] = relu(e1[a] @ W2 + b2)
// grid = (A, 4): a block owns 64 output columns of one action; its 256 threads = 64 columns x 4 K slices
// (the 256-long dot products are latency-bound, so the reduction is split and combined through shared memory)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) emb_forward_kernel(const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ w2, const float* __restrict__ b2,
                                                           float* __restrict__ e1, float* __restrict__ table) {
  kernel_prologue();
  __shared__ float se[Geo::EMB];
  __shared__ float part[4][64];
  const int a = blockIdx.x, tid = threadIdx.x;
  const float v = fmaxf(w1[a * Geo::EMB + tid] + b1[tid], 0.f);
  se[tid] = v;
  if (blockIdx.y == 0) e1[a * Geo::EMB + tid] = v;
  __syncthreads();
  const int c = tid & 63, ks = tid >> 6;
  const int j = blockIdx.y * 64 + c;
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 8
  for (int k = ks * 64; k < ks * 64 + 64; k += 2) {
    acc0 = fmaf(se[k], __ldg(w2 + k * Geo::EMB + j), acc0);
    acc1 = fmaf(se[k + 1], __ldg(w2 + (k + 1) * Geo::EMB + j), acc1);
  }
  part[ks][c] = acc0 + acc1;
  __syncthreads();
  if (tid < 64) {
    const float s = (part[0][tid] + part[1][tid]) + (part[2][tid] + part[3][tid]);
    table[a * Geo::EMB + j] = fmaxf(s + b2[j], 0.f);
  }
}

int emb_forward(cudaStream_t s, const float* w1, const float* b1, const float* w2, const float* b2, float* e1,
                float* table, int A) {
  DRL_CUDA_CHECK((launch_k(emb_forward_kernel, dim3(A, 4), 256, 0, s, w1, b1, w2, b2, e1, table)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// LSTM gates forward (model/impala_actor_critic.py:18-25; TF 1.14 LSTMCell):
//   z = sum_s zpart[s] + b ; i,j,f,o = split(z,4)
//   c1 = sigmoid(f + 1) * c0 + sigmoid(i) * tanh(j) ; h1 = sigmoid(o) * tanh(c1)
// thread per (row m, unit u); c0 is batch-major [B,T,256].
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) lstm_gates_forward_kernel(
    const float* __restrict__ zpart, int nsplit, size_t split_stride, const float* __restrict__ bias,
    const float* __restrict__ c0, float* __restrict__ gates, float* __restrict__ c1, float* __restrict__ tc1,
    float* __restrict__ h1, int M, int B, int T) {
  kernel_prologue();
  const int m = blockIdx.x, u = threadIdx.x;
  if (m >= M) return;
  const int t = m / B, b = m - t * B;
  const size_t src = (size_t)(b * T + t) * Geo::L + u;
  float z[4];
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    float acc = 0.f;
    for (int s = 0; s < nsplit; ++s) acc += zpart[s * split_stride + (size_t)m * Geo::G4 + g * Geo::L + u];
    z[g] = acc + bias[g * Geo::L + u];
  }
  const float si = sigmoidf_acc(z[0]);
  const float tj = tanhf(z[1]);
  const float sf = sigmoidf_acc(z[2] + 1.0f);
  const float so = sigmoidf_acc(z[3]);
  const float c = sf * c0[src] + si * tj;
  const float tc = tanhf(c);
  const size_t o = (size_t)m * Geo::L + u;
  float* g = gates + (size_t)m * Geo::G4;
  g[u] = si; g[Geo::L + u] = tj; g[2 * Geo::L + u] = sf; g[3 * Geo::L + u] = so;
  c1[o] = c; tc1[o] = tc; h1[o] = so * tc;
}

int lstm_gates_forward(cudaStream_t s, const float* zpart, int nsplit, const float* bias, const float* c0,
                       float* gates, float* c1, float* tc1, float* h1, int M, int B, int T) {
  DRL_CUDA_CHECK((launch_k(lstm_gates_forward_kernel, M, 256, 0, s, zpart, nsplit, (size_t)M * Geo::G4, bias, c0, gates, c1, tc1, h1, M, B,
                                              T)));
  return DRL_OK;
}

// backward of the cell for rows m < Mb:  dh = dh_part[0] + dh_part[1]
//   do = dh*tc*so(1-so) ; dc = dh*so*(1-tc^2) ; di = dc*tj*si(1-si) ; dj = dc*si*(1-tj^2) ; df = dc*c0*sf(1-sf)
__global__ void __launch_bounds__(256) lstm_gates_backward_kernel(
    const float* __restrict__ dh_part, size_t part_stride, const float* __restrict__ gates,
    const float* __restrict__ tc1, const float* __restrict__ c0, float* __restrict__ dz, int Mb, int B, int T) {
  kernel_prologue();
  const int m = blockIdx.x, u = threadIdx.x;
  if (m >= Mb) return;
  const int t = m / B, b = m - t * B;
  const size_t o = (size_t)m * Geo::L + u;
  const float dh = dh_part[o] + dh_part[part_stride + o];
  const float* g = gates + (size_t)m * Geo::G4;
  const float si = g[u], tj = g[Geo::L + u], sf = g[2 * Geo::L + u], so = g[3 * Geo::L + u];
  const float tc = tc1[o];
  const float cprev = c0[(size_t)(b * T + t) * Geo::L + u];
  const float d_o = dh * tc * so * (1.f - so);
  const float dc = dh * so * (1.f - tc * tc);
  float* d = dz + (size_t)m * Geo::G4;
  d[u] = dc * tj * si * (1.f - si);
  d[Geo::L + u] = dc * si * (1.f - tj * tj);
  d[2 * Geo::L + u] = dc * cprev * sf * (1.f - sf);
  d[3 * Geo::L + u] = d_o;
}

int lstm_gates_backward(cudaStream_t s, const float* dh_part, size_t part_stride, const float* gates,
                        const float* tc1, const float* c0, float* dz, int Mb, int B, int T) {
  DRL_CUDA_CHECK((launch_k(lstm_gates_backward_kernel, Mb, 256, 0, s, dh_part, part_stride, gates, tc1, c0, dz, Mb, B, T)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// Output layers (model/impala_actor_critic.py:40-41): logits = hid2_a @ W5 + b5 (256 -> A),
// policy = softmax(logits), value = hid2_c @ w8 + b8.  One warp per row; lanes split K.
// ------------------------------------------------------------------------------------------
constexpr int kMaxA = 32;

__global__ void __launch_bounds__(128) heads_out_forward_kernel(
    const float* __restrict__ ha, const float* __restrict__ hc, const float* __restrict__ w5,
    const float* __restrict__ b5, const float* __restrict__ w8, const float* __restrict__ b8,
    float* __restrict__ logits, float* __restrict__ policy, float* __restrict__ value, int M, int A) {
  kernel_prologue();
  extern __shared__ __align__(16) float sw[];   // W5 [256*A] then w8 [256]
  // Weight staging with every load in flight at once: as a scalar loop this was 36 loads per thread that the compiler
  // issued four at a time -- nine dependent round trips to L2 (~6 us) in front of 2 us of arithmetic.
  if ((reinterpret_cast<uintptr_t>(w5) & 15) == 0 && (reinterpret_cast<uintptr_t>(w8) & 15) == 0) {
    const float4* w54 = reinterpret_cast<const float4*>(w5);
    const int n4 = Geo::HID * A / 4;                 // HID = 256: a multiple of 4 for every A
    float4 tmp[kMaxA / 2];                           // n4 / 128 threads = A / 2 <= 16 per thread
#pragma unroll
    for (int j = 0; j < kMaxA / 2; ++j) {
      const int i = threadIdx.x + j * 128;
      if (i < n4) tmp[j] = __ldg(w54 + i);
    }
    float4 t8 = zero4();
    if (threadIdx.x < Geo::HID / 4) t8 = __ldg(reinterpret_cast<const float4*>(w8) + threadIdx.x);
#pragma unroll
    for (int j = 0; j < kMaxA / 2; ++j) {
      const int i = threadIdx.x + j * 128;
      if (i < n4) reinterpret_cast<float4*>(sw)[i] = tmp[j];
    }
    if (threadIdx.x < Geo::HID / 4) reinterpret_cast<float4*>(sw + Geo::HID * A)[threadIdx.x] = t8;
  } else {
    for (int i = threadIdx.x; i < Geo::HID * A; i += blockDim.x) sw[i] = w5[i];
    for (int i = threadIdx.x; i < Geo::HID; i += blockDim.x) sw[Geo::HID * A + i] = w8[i];
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * 4 + warp;
  __syncthreads();
  if (m >= M) return;
  float acc[kMaxA];
#pragma unroll
  for (int a = 0; a < kMaxA; ++a) acc[a] = 0.f;
  float vacc = 0.f;
  // the row's 2 x 256 activations first: 16 independent loads in flight instead of 8 dependent round trips to L2
  float xa[Geo::HID / 32], xc[Geo::HID / 32];
#pragma unroll
  for (int i = 0; i < Geo::HID / 32; ++i) {
    xa[i] = ha[(size_t)m * Geo::HID + lane + 32 * i];
    xc[i] = hc[(size_t)m * Geo::HID + lane + 32 * i];
  }
#pragma unroll
  for (int i = 0; i < Geo::HID / 32; ++i) {
    const int k = lane + 32 * i;
    vacc = fmaf(xc[i], sw[Geo::HID * A + k], vacc);
#pragma unroll
    for (int a = 0; a < kMaxA; ++a)
      if (a < A) acc[a] = fmaf(xa[i], sw[k * A + a], acc[a]);
  }
  vacc = warp_sum(vacc);
  float mine = -INFINITY;   // lane a keeps logit a
  float mx = -INFINITY;
#pragma unroll
  for (int a = 0; a < kMaxA; ++a) {
    if (a < A) {
      const float l = warp_sum(acc[a]) + b5[a];
      mx = fmaxf(mx, l);
      if (lane == a) mine = l;
    }
  }
  const float e = (lane < A) ? expf(mine - mx) : 0.f;
  const float sum = warp_sum(e);
  if (lane < A) {
    logits[(size_t)m * A + lane] = mine;
    policy[(size_t)m * A + lane] = e / sum;
  }
  if (lane == 0) value[m] = vacc + b8[0];
}

int heads_out_forward(cudaStream_t s, const float* ha, const float* hc, const float* w5, const float* b5,
                      const float* w8, const float* b8, float* logits, float* policy, float* value, int M, int A) {
  if (A > kMaxA) { set_error("num_action %d > %d unsupported", A, kMaxA); return DRL_ERR_INVALID; }
  const size_t smem = (size_t)(Geo::HID * A + Geo::HID) * sizeof(float);
  DRL_CUDA_CHECK((launch_k(heads_out_forward_kernel, cdiv(M, 4), 128, smem, s, ha, hc, w5, b5, w8, b8, logits, policy, value, M, A)));
  return DRL_OK;
}

// dhid2_a[m,k] = relu'(hid2_a) * sum_a dlogits[m,a] W5[k,a] ; dhid2_c[m,k] = relu'(hid2_c) * dv[m] * w8[k]
// grid = Mb blocks, 256 threads (k).  dlogits / dv have row stride 32.
__global__ void __launch_bounds__(256) heads_out_backward_kernel(
    const float* __restrict__ dlogits, const float* __restrict__ dv, const float* __restrict__ w5,
    const float* __restrict__ w8, const float* __restrict__ ha, const float* __restrict__ hc,
    float* __restrict__ dha, float* __restrict__ dhc, int Mb, int A) {
  kernel_prologue();
  __shared__ float sd[kMaxA];
  __shared__ float sdv;
  const int m = blockIdx.x, k = threadIdx.x;
  if (k < A) sd[k] = dlogits[(size_t)m * 32 + k];
  if (k == 0) sdv = dv[(size_t)m * 32];
  __syncthreads();
  float acc = 0.f;
  for (int a = 0; a < A; ++a) acc = fmaf(sd[a], __ldg(w5 + k * A + a), acc);
  const size_t o = (size_t)m * Geo::HID + k;
  dha[o] = (ha[o] > 0.f) ? acc : 0.f;
  dhc[o] = (hc[o] > 0.f) ? sdv * __ldg(w8 + k) : 0.f;
}

int heads_out_backward(cudaStream_t s, const float* dlogits, const float* dv, const float* w5, const float* w8,
                       const float* ha, const float* hc, float* dha, float* dhc, int Mb, int A) {
  DRL_CUDA_CHECK((launch_k(heads_out_backward_kernel, Mb, 256, 0, s, dlogits, dv, w5, w8, ha, hc, dha, dhc, Mb, A)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// Action-embedding backward.  All rows with the same previous action share the same masks, so
// the per-row gradients are first summed per action (segment sum) and then pushed through the
// A-row MLP once (linear in the upstream gradient, so this equals the per-row backward summed).
// ------------------------------------------------------------------------------------------
// (1a) part[c][a][j] = sum_{m in row chunk c, pa[m]==a} du[m,j]                       grid (A, kEmbChunks), 256 threads
constexpr int kEmbChunks = 16;
__global__ void __launch_bounds__(256) emb_segsum_kernel(const float* __restrict__ du, const int32_t* __restrict__ pa,
                                                          float* __restrict__ part, int Mb, int B, int T, int A) {
  kernel_prologue();
  const int a = blockIdx.x, c = blockIdx.y, j = threadIdx.x;
  const int per = (Mb + kEmbChunks - 1) / kEmbChunks;
  const int lo = c * per, hi = min(Mb, lo + per);
  float acc = 0.f;
  for (int m = lo; m < hi; ++m) {
    const int t = m / B, b = m - t * B;
    if (__ldg(pa + b * T + t) == a) acc += du[(size_t)m * Geo::EMB + j];
  }
  part[((size_t)c * A + a) * Geo::EMB + j] = acc;
}
// (1b) dpre2[a,j] = relu'(table[a,j]) * sum_c part[c][a][j]   (fixed order)           grid A, 256 threads
__global__ void __launch_bounds__(256) emb_dpre2_kernel(const float* __restrict__ part, const float* __restrict__ table,
                                                         float* __restrict__ dpre2, int A) {
  kernel_prologue();
  const int a = blockIdx.x, j = threadIdx.x;
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < kEmbChunks; ++c) acc += part[((size_t)c * A + a) * Geo::EMB + j];
  dpre2[a * Geo::EMB + j] = (table[a * Geo::EMB + j] > 0.f) ? acc : 0.f;
}
// (2) g_w2[k,j] = sum_a e1[a,k] dpre2[a,j] ; g_b2[j] = sum_a dpre2[a,j]             grid 256 (k), 256 threads (j)
__global__ void __launch_bounds__(256) emb_bwd2_kernel(const float* __restrict__ e1, const float* __restrict__ dpre2,
                                                        float* __restrict__ g_w2, float* __restrict__ g_b2, int A) {
  kernel_prologue();
  const int k = blockIdx.x, j = threadIdx.x;
  float acc = 0.f, bs = 0.f;
  for (int a = 0; a < A; ++a) {
    const float d = dpre2[a * Geo::EMB + j];
    acc = fmaf(__ldg(e1 + a * Geo::EMB + k), d, acc);
    bs += d;
  }
  g_w2[k * Geo::EMB + j] = acc;
  if (k == 0) g_b2[j] = bs;
}
// (3) dpre1[a,k] = relu'(e1[a,k]) * sum_j dpre2[a,j] W2[k,j] ; g_w1[a,k] = dpre1[a,k] ; g_b1[k] = sum_a dpre1[a,k]
//     grid 32 blocks x 8 warps; one warp per k, lanes over j.
__global__ void __launch_bounds__(256) emb_bwd1_kernel(const float* __restrict__ e1, const float* __restrict__ dpre2,
                                                        const float* __restrict__ w2, float* __restrict__ dpre1,
                                                        float* __restrict__ g_w1, float* __restrict__ g_b1, int A) {
  kernel_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.x * 8 + warp;
  float w[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) w[i] = w2[(size_t)k * Geo::EMB + lane + 32 * i];
  float bs = 0.f;
  for (int a = 0; a < A; ++a) {
    float p = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) p = fmaf(dpre2[a * Geo::EMB + lane + 32 * i], w[i], p);
    p = warp_sum(p);
    const float d = (e1[a * Geo::EMB + k] > 0.f) ? p : 0.f;
    if (lane == 0) {
      dpre1[a * Geo::EMB + k] = d;
      g_w1[a * Geo::EMB + k] = d;
    }
    bs += d;
  }
  if (lane == 0) g_b1[k] = bs;
}

int emb_backward(cudaStream_t s, const float* du, const int32_t* pa, const float* e1, const float* table,
                 const float* w2, float* dpre2, float* dpre1, float* g_w1, float* g_b1, float* g_w2, float* g_b2,
                 float* scratch, int Mb, int B, int T, int A) {
  // scratch: >= kEmbChunks * A * 256 floats (the split-K partial buffer, idle at this point of the step)
  DRL_CUDA_CHECK((launch_k(emb_segsum_kernel, dim3(A, kEmbChunks), 256, 0, s, du, pa, scratch, Mb, B, T, A)));
  DRL_CUDA_CHECK((launch_k(emb_dpre2_kernel, A, 256, 0, s, scratch, table, dpre2, A)));
  DRL_CUDA_CHECK((launch_k(emb_bwd2_kernel, Geo::EMB, 256, 0, s, e1, dpre2, g_w2, g_b2, A)));
  DRL_CUDA_CHECK((launch_k(emb_bwd1_kernel, Geo::EMB / 8, 256, 0, s, e1, dpre2, w2, dpre1, g_w1, g_b1, A)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// col2im + ReLU mask: second half of the convolution data gradient in its "dCol" form
//   dCol[(img,oy,ox), (ky,kx,ci)] = sum_co dY[img,oy,ox,co] W[ky,kx,ci,co]         (one plain GEMM, K = CO)
//   dX[img,y,x,ci] = relu'(act) * sum_{ky,kx : (y-ky)%S == 0, (x-kx)%S == 0, oy,ox in range} dCol[(img,oy,ox),(ky,kx,ci)]
// One thread per (pixel, 4 channels): <= (KH/S)*(KW/S) float4 reads, deterministic (a gather, no atomics).
// ------------------------------------------------------------------------------------------
template <int IH, int IW, int CI, int OH, int OW, int KH, int KW, int S>
__global__ void __launch_bounds__(256) col2im_relu_kernel(const float* __restrict__ dcol,
                                                           const float* __restrict__ act, float* __restrict__ dx,
                                                           int nimg) {
  kernel_prologue();
  constexpr int C4 = CI / 4, NCOL = KH * KW * CI;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)nimg * IH * IW * C4;
  if (idx >= total) return;
  const int c4 = (int)(idx % C4);
  const long long pix = idx / C4;
  const int x = (int)(pix % IW);
  const int y = (int)((pix / IW) % IH);
  const int img = (int)(pix / (IW * IH));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int jy = 0; jy < KH / S; ++jy) {
    const int ky = (y % S) + jy * S;
    const int oy = (y - ky) / S;
    if (oy < 0 || oy >= OH) continue;
#pragma unroll
    for (int jx = 0; jx < KW / S; ++jx) {
      const int kx = (x % S) + jx * S;
      const int ox = (x - kx) / S;
      if (ox < 0 || ox >= OW) continue;
      const float4 v = __ldg(reinterpret_cast<const float4*>(
          dcol + ((size_t)(img * OH + oy) * OW + ox) * NCOL + (ky * KW + kx) * CI + c4 * 4));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  const size_t o = (size_t)pix * CI + c4 * 4;
  const float4 a = __ldg(reinterpret_cast<const float4*>(act + o));
  *reinterpret_cast<float4*>(dx + o) = make_float4(a.x > 0.f ? acc.x : 0.f, a.y > 0.f ? acc.y : 0.f,
                                                   a.z > 0.f ? acc.z : 0.f, a.w > 0.f ? acc.w : 0.f);
}

int col2im_conv3(cudaStream_t s, const float* dcol, const float* a2, float* da2, int nimg) {
  const long long total = (long long)nimg * 9 * 9 * 16;
  DRL_CUDA_CHECK((launch_k(col2im_relu_kernel<9, 9, 64, 7, 7, 3, 3, 1>, (unsigned)cdiv64(total, 256), 256, 0, s, dcol, a2, da2, nimg)));
  return DRL_OK;
}
int col2im_conv2(cudaStream_t s, const float* dcol, const float* a1, float* da1, int nimg) {
  const long long total = (long long)nimg * 20 * 20 * 8;
  DRL_CUDA_CHECK((launch_k(col2im_relu_kernel<20, 20, 32, 9, 9, 4, 4, 2>, (unsigned)cdiv64(total, 256), 256, 0, s, dcol, a1, da1, nimg)));
  return DRL_OK;
}

// ------------------------------------------------------------------------------------------
// out[j] = sum_z part[z*slab + j]   (deterministic split-K reduction)
// ------------------------------------------------------------------------------------------
// 256 threads = 32 consecutive outputs (one 128-byte line per slab) x 8 slab groups: group g sums slabs g, g+8, ... with
// four independent accumulators, the eight group sums are then added in the fixed order 0..7 -- the serial chain per
// thread is nsplit/8 loads instead of nsplit (many per-CTA slabs: fewer dependent loads on the critical path).
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ part, size_t slab, int nsplit,
                                                             float* __restrict__ out, size_t n) {
  kernel_prologue();
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const size_t j = (size_t)blockIdx.x * 32 + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (j < n) {
    int z = g;
    for (; z + 24 < nsplit; z += 32) {
      a0 += part[(size_t)z * slab + j];
      a1 += part[(size_t)(z + 8) * slab + j];
      a2 += part[(size_t)(z + 16) * slab + j];
      a3 += part[(size_t)(z + 24) * slab + j];
    }
    for (; z < nsplit; z += 8) a0 += part[(size_t)z * slab + j];
  }
  red[g][lane] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (g == 0 && j < n) {
    float v = red[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) v += red[k][lane];
    out[j] = v;
  }
}

int splitk_reduce(cudaStream_t s, const float* part, size_t slab, int nsplit, float* out, size_t n) {
  DRL_CUDA_CHECK((launch_k(splitk_reduce_kernel, (unsigned)cdiv64((int64_t)n, 32), 256, 0, s, part, slab, nsplit, out, n)));
  return DRL_OK;
}

}  // namespace drl
