// l2_bulk_bw.cu -- how fast can all SMs pull an L2-resident operand into shared memory?
//   mode 0: cp.async.bulk (global -> shared, mbarrier complete_tx), CHUNK bytes per copy, 2..4 stages in flight
//   mode 1: LDG.128 by 256 threads per CTA (registers only, no shared-memory store)
// The window (default 16 MB) is re-read many times, so after the first pass every byte comes from L2.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o l2_bulk_bw l2_bulk_bw.cu
// Usage: ./l2_bulk_bw [window_MB=16] [chunk_KB=32] [stages=3] [ctas_per_sm=1]
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, int n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t ph) {
  asm volatile("{\n.reg .pred p;\nW: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D;\nbra W;\nD:\n}" ::"r"(smem_u32(b)), "r"(ph) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory");
}

__global__ void bulk_kernel(const uint8_t* win, size_t win_bytes, int chunk, int stages, int iters, unsigned long long* sink) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t bar[8];
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const size_t nchunks = win_bytes / chunk;
    size_t c = ((size_t)blockIdx.x * 7919u) % nchunks;
    for (int i = 0; i < iters + stages; ++i) {
      const int s = i % stages;
      if (i >= stages) mbar_wait(&bar[s], ((i / stages) - 1) & 1);
      if (i < iters) {
        mbar_expect(&bar[s], chunk);
        bulk_g2s(smem + (size_t)s * chunk, win + c * chunk, chunk, &bar[s]);
        c += gridDim.x; if (c >= nchunks) c -= nchunks; if (c >= nchunks) c %= nchunks;
      }
    }
    if (sink && smem[0] == 123 && smem[chunk] == 77) *sink = 1;
  }
}

__global__ void ldg_kernel(const uint4* win, size_t n16, int iters, unsigned long long* sink) {
  // every CTA streams `iters` x (blockDim * 4) 16-byte words, 4 independent loads in flight per thread
  size_t idx = ((size_t)blockIdx.x * 7919u * 1024u + threadIdx.x) % n16;
  uint4 acc = make_uint4(0, 0, 0, 0);
  const size_t stride = (size_t)gridDim.x * blockDim.x * 4;
  for (int i = 0; i < iters; ++i) {
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { size_t k = idx + (size_t)j * blockDim.x; if (k >= n16) k -= n16; v[j] = __ldcg(win + k); }
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc.x ^= v[j].x; acc.y ^= v[j].y; acc.z ^= v[j].z; acc.w ^= v[j].w; }
    idx += stride; while (idx >= n16) idx -= n16;
  }
  if (acc.x == 0x12345678u && acc.y == 1u) *sink = acc.z;
}

int main(int argc, char** argv) {
  const int win_mb = argc > 1 ? atoi(argv[1]) : 16;
  const int chunk = (argc > 2 ? atoi(argv[2]) : 32) * 1024;
  const int stages = argc > 3 ? atoi(argv[3]) : 3;
  const int per_sm = argc > 4 ? atoi(argv[4]) : 1;
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  const size_t win_bytes = (size_t)win_mb << 20;
  uint8_t* win; CK(cudaMalloc(&win, win_bytes)); CK(cudaMemset(win, 1, win_bytes));
  unsigned long long* sink; CK(cudaMalloc(&sink, 8));
  const int grid = p.multiProcessorCount * per_sm;
  const size_t smem = (size_t)stages * chunk;
  CK(cudaFuncSetAttribute(bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int iters = 400;
  for (int rep = 0; rep < 3; ++rep) {
    CK(cudaEventRecord(e0));
    bulk_kernel<<<grid, 32, smem>>>(win, win_bytes, chunk, stages, iters, sink);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    const double bytes = (double)grid * iters * chunk;
    printf("bulk  window %d MB chunk %d KB stages %d ctas/sm %d : %.3f ms  %.2f TB/s  (%.1f B/clk/SM @1.9GHz)\n", win_mb, chunk >> 10, stages,
           per_sm, ms, bytes / ms * 1e-9, bytes / ms * 1e-6 / p.multiProcessorCount / 1.9e3);
  }
  for (int rep = 0; rep < 3; ++rep) {
    const int it2 = 200;
    CK(cudaEventRecord(e0));
    ldg_kernel<<<grid * 2, 256>>>((const uint4*)win, win_bytes / 16, it2, sink);
    CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    const double bytes = (double)grid * 2 * it2 * 256 * 4 * 16;
    printf("ldg128 window %d MB, %d CTAs x 256 thr, 4 loads in flight : %.3f ms  %.2f TB/s\n", win_mb, grid * 2, ms, bytes / ms * 1e-9);
  }
  return 0;
}
