// common.cuh -- error handling and small device helpers shared by all kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

#include "../../include/drl_b200.h"

namespace drl {

// thread-local last-error text behind drl_last_error()
void set_error(const char* fmt, ...);
const char* get_error();

#define DRL_CUDA_CHECK(expr)                                                          \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      ::drl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),        \
                       __FILE__, __LINE__);                                           \
      return DRL_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

#define DRL_CHECK_LAUNCH()                                                            \
  do {                                                                                \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess) {                                                          \
      ::drl::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),    \
                       __FILE__, __LINE__);                                           \
      return DRL_ERR_CUDA;                                                            \
    }                                                                                 \
  } while (0)

#define DRL_TRY(expr)              \
  do {                             \
    int _r = (expr);               \
    if (_r != DRL_OK) return _r;   \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- kernel start-time trace ----------------------------------------------------------
// Every kernel of the learners starts with kernel_prologue().  When the trace is armed (drl_debug_trace), CTA (0,0,0)
// appends {globaltimer ns, grid size << 32 | block size} to a device buffer, which gives the true kernel timeline inside a
// CUDA-graph replay (both streams), something CUDA events cannot do without serialising the graph.  The pointer is a
// per-translation-unit device global (no relocatable device code); every TU registers a setter at load time.
static __device__ unsigned long long* g_trace_tu = nullptr;
__device__ __forceinline__ void kernel_prologue() {
  unsigned long long* tr = g_trace_tu;
  if (tr != nullptr && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    const unsigned long long i = atomicAdd(tr, 1ULL);
    if (i < 4000ULL) {
      tr[1 + 2 * i] = t;
      tr[2 + 2 * i] = ((unsigned long long)(gridDim.x * gridDim.y * gridDim.z) << 32) | (unsigned long long)blockDim.x;
    }
  }
}
typedef void (*TraceSetter)(unsigned long long*);
int register_trace_setter(TraceSetter f);            // learner_core.cu
static void trace_set_tu(unsigned long long* p) { cudaMemcpyToSymbol(g_trace_tu, &p, sizeof(p)); }
static const int g_trace_registered = register_trace_setter(&trace_set_tu);

template <class... KA, class... A>
inline cudaError_t launch_k(void (*kern)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KA>(args)...);
}

// ---- device helpers ------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// 1 / (1 + e^-x) with the approximate-reciprocal division (<= 2 ulp): the IEEE division's FCHK + slow-path subroutine costs
// hundreds of cycles per element in the gate kernels (see div255 in loaders.cuh for the measurement)
__device__ __forceinline__ float sigmoidf_acc(float x) { return __fdividef(1.0f, 1.0f + expf(-x)); }

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// Geometry of the reference network (model/impala_actor_critic.py:5-10): fixed at compile time.
struct Geo {
  static constexpr int IH = 84, IW = 84, IC = 4;
  static constexpr int C1H = 20, C1W = 20, C1C = 32;   // conv 8x8 s4
  static constexpr int C2H = 9, C2W = 9, C2C = 64;     // conv 4x4 s2
  static constexpr int C3H = 7, C3W = 7, C3C = 64;     // conv 3x3 s1
  static constexpr int FLAT = C3H * C3W * C3C;         // 3136
  static constexpr int EMB = 256;                      // action-embedding width
  static constexpr int L = 256;                        // lstm units
  static constexpr int XK = FLAT + EMB + L;            // 3648 = LSTM kernel rows
  static constexpr int G4 = 4 * L;                     // 1024 gate columns
  static constexpr int HID = 256;                      // head hidden width
  static constexpr int FRAME = IH * IW * IC;           // 28224 bytes
};

}  // namespace drl
