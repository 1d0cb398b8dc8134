// bulk_gemm_feed.cu -- what limits the operand feed of the bulk-fed LSTM GEMMs (csrc/gemm_bulk16.cuh)?
// Replays ONLY the loader of lstm_dgrad / lstm_wgrad / lstm_fwd (no MMAs): a grid of (MT x NT) CTAs, each streaming KT K tiles
// of [A tile | B tile] into a STAGES-deep shared-memory ring with cp.async.bulk, a consumer thread "using" a stage for
// `hold` ns before it frees it.  Variants: tiles SHARED between CTAs as in the GEMM (A tile by all CTAs of an m row, B tile
// by all CTAs of an n column) or PRIVATE per CTA; one or two issuing lanes; chunked copies.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o bulk_gemm_feed bulk_gemm_feed.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, int n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n)); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t ph) {
  asm volatile("{\n.reg .pred p;\nW: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D;\nbra W;\nD:\n}" ::"r"(smem_u32(b)), "r"(ph) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory");
}

struct P {
  const uint8_t *a, *b;
  int MT, NT, KT, a_bytes, b_bytes, stages, shared, lanes, split, hold_ns;
};

__global__ void feed_kernel(P p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ uint64_t full[8], empty[8];
  const int stage_bytes = p.a_bytes + p.b_bytes;
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full[s], p.lanes); mbar_init(&empty[s], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int mt = blockIdx.x % p.MT, nt = blockIdx.x / p.MT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t a_row = p.shared ? (size_t)mt : (size_t)blockIdx.x, b_row = p.shared ? (size_t)nt : (size_t)blockIdx.x;
  if (warp < p.lanes && lane == 0) {
    for (int t = 0; t < p.KT; ++t) {
      const int s = t % p.stages;
      mbar_wait(&empty[s], ((t / p.stages) & 1) ^ 1);
      uint8_t* st = smem + (size_t)s * stage_bytes;
      const uint8_t* asrc = p.a + (a_row * p.KT + t) * (size_t)p.a_bytes;
      const uint8_t* bsrc = p.b + (b_row * p.KT + t) * (size_t)p.b_bytes;
      if (p.lanes == 1) {
        mbar_expect(&full[s], stage_bytes);
        for (int c = 0; c < p.split; ++c) bulk_g2s(st + c * (p.a_bytes / p.split), asrc + c * (p.a_bytes / p.split), p.a_bytes / p.split, &full[s]);
        for (int c = 0; c < p.split; ++c) bulk_g2s(st + p.a_bytes + c * (p.b_bytes / p.split), bsrc + c * (p.b_bytes / p.split), p.b_bytes / p.split, &full[s]);
      } else if (warp == 0) {
        mbar_expect(&full[s], p.a_bytes);
        bulk_g2s(st, asrc, p.a_bytes, &full[s]);
      } else {
        mbar_expect(&full[s], p.b_bytes);
        bulk_g2s(st + p.a_bytes, bsrc, p.b_bytes, &full[s]);
      }
    }
  } else if (warp == 2 && lane == 0) {
    for (int t = 0; t < p.KT; ++t) {
      const int s = t % p.stages;
      mbar_wait(&full[s], (t / p.stages) & 1);
      if (p.hold_ns) __nanosleep(p.hold_ns);
      mbar_arrive(&empty[s]);
    }
  }
}

int main(int argc, char** argv) {
  // defaults = lstm_dgrad: 5 x 27 CTAs, 16 K tiles, A 32 KB + B 32 KB, 3 stages
  P p{};
  p.MT = argc > 1 ? atoi(argv[1]) : 5; p.NT = argc > 2 ? atoi(argv[2]) : 27; p.KT = argc > 3 ? atoi(argv[3]) : 16;
  p.a_bytes = (argc > 4 ? atoi(argv[4]) : 32) * 1024; p.b_bytes = (argc > 5 ? atoi(argv[5]) : 32) * 1024;
  p.stages = argc > 6 ? atoi(argv[6]) : 3; p.shared = argc > 7 ? atoi(argv[7]) : 1; p.lanes = argc > 8 ? atoi(argv[8]) : 1;
  p.split = argc > 9 ? atoi(argv[9]) : 1; p.hold_ns = argc > 10 ? atoi(argv[10]) : 0;
  const int grid = p.MT * p.NT;
  const size_t a_total = (size_t)(p.shared ? p.MT : grid) * p.KT * p.a_bytes, b_total = (size_t)(p.shared ? p.NT : grid) * p.KT * p.b_bytes;
  uint8_t *a, *b, *flush; CK(cudaMalloc(&a, a_total)); CK(cudaMalloc(&b, b_total)); CK(cudaMalloc(&flush, 256u << 20));
  const size_t smem = (size_t)p.stages * (p.a_bytes + p.b_bytes);
  CK(cudaFuncSetAttribute(feed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  p.a = a; p.b = b;
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (int mode = 0; mode < 3; ++mode) {   // 0: operands just written (as after the image kernels), 1: warm (second launch), 2: L2 flushed
    float best = 1e9f, sum = 0.f;
    for (int rep = 0; rep < 5; ++rep) {
      if (mode == 0) { CK(cudaMemsetAsync(a, rep + 1, a_total)); CK(cudaMemsetAsync(b, rep + 2, b_total)); }
      if (mode == 2) CK(cudaMemsetAsync(flush, rep, 256u << 20));
      CK(cudaEventRecord(e0));
      feed_kernel<<<grid, 96, smem>>>(p);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      if (rep) { best = ms < best ? ms : best; sum += ms; }
    }
    const double bytes = (double)grid * p.KT * (p.a_bytes + p.b_bytes);
    printf("grid %dx%d KT %d A %dK B %dK stages %d shared %d lanes %d split %d hold %d ns | %s: best %.1f us avg %.1f us  %.2f TB/s (%.0f MB)\n",
           p.MT, p.NT, p.KT, p.a_bytes >> 10, p.b_bytes >> 10, p.stages, p.shared, p.lanes, p.split, p.hold_ns,
           mode == 0 ? "fresh" : mode == 1 ? "warm " : "flush", best * 1e3, sum / 4 * 1e3, bytes / best * 1e-9, bytes * 1e-6);
  }
  return 0;
}
