// tma_box_bw.cu -- throughput of TMA tensor loads (cp.async.bulk.tensor, SWIZZLE_128B) whose box is made of many
// 128-byte rows, the shape an im2col tile of an NHWC activation has, against a plain 2-D box and a linear bulk copy
// of the same size.  One thread per CTA keeps `stages` loads in flight; the tensor (16 MB) is L2 resident.
//   mode 0: 4-D box {32, W, W, 1} over dims {32, W, W, N} with strides {sx*128 B, sy*ROWPITCH, IMG} (conv gather)
//   mode 1: 2-D box {32, W*W} over a dense [rows, 32] fp32 matrix (contiguous 128-byte rows)
//   mode 2: cp.async.bulk of W*W*128 contiguous bytes
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tma_box_bw tma_box_bw.cu
// Usage: ./tma_box_bw [W=9] [stride=2] [stages=4] [ctas_per_sm=1]
#include <cuda.h>
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

struct Maps { CUtensorMap m4, m2; };

__global__ void tma_kernel(const __grid_constant__ Maps maps, const uint8_t* lin, int mode, int nimg, int box_bytes, int stages,
                           int iters, unsigned long long* sink) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  __shared__ uint64_t bar[8];
  const int slot = (box_bytes + 1023) / 1024 * 1024;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(&bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int img = (blockIdx.x * 37) % nimg;
    for (int i = 0; i < iters + stages; ++i) {
      const int s = i % stages;
      if (i >= stages) mbar_wait(&bar[s], ((i / stages) - 1) & 1);
      if (i < iters) {
        mbar_expect(&bar[s], box_bytes);
        uint8_t* dst = smem + (size_t)s * slot;
        if (mode == 0) {
          asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                       ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(&maps.m4)), "r"(0), "r"(0), "r"(0), "r"(img), "r"(smem_u32(&bar[s])) : "memory");
        } else if (mode == 1) {
          asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                       ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(&maps.m2)), "r"(0), "r"(img * (box_bytes / 128)), "r"(smem_u32(&bar[s])) : "memory");
        } else {
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                       ::"r"(smem_u32(dst)), "l"(lin + (size_t)img * box_bytes), "r"(box_bytes), "r"(smem_u32(&bar[s])) : "memory");
        }
        img += gridDim.x; while (img >= nimg) img -= nimg;
      }
    }
    if (sink && smem[5] == 123 && smem[77] == 9) *sink = 1;
  }
}

typedef CUresult (*EncFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                          const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                          CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main(int argc, char** argv) {
  const int W = argc > 1 ? atoi(argv[1]) : 9;
  const int stride = argc > 2 ? atoi(argv[2]) : 2;
  const int stages = argc > 3 ? atoi(argv[3]) : 4;
  const int per_sm = argc > 4 ? atoi(argv[4]) : 1;
  const int IH = stride * (W - 1) + 4;                 // input rows/cols of one image (like conv2: 20 for W=9, s=2)
  const size_t img_bytes = (size_t)IH * IH * 128;
  const int nimg = (int)((16u << 20) / img_bytes);
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  uint8_t* buf; CK(cudaMalloc(&buf, (size_t)nimg * img_bytes + 4096)); CK(cudaMemset(buf, 1, (size_t)nimg * img_bytes));
  unsigned long long* sink; CK(cudaMalloc(&sink, 8));
  void* fp = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
  EncFn enc = (EncFn)fp;
  Maps maps;
  {
    const cuuint64_t dims[4] = {32, (cuuint64_t)W, (cuuint64_t)W, (cuuint64_t)nimg};
    const cuuint64_t strides[3] = {(cuuint64_t)stride * 128, (cuuint64_t)stride * IH * 128, (cuuint64_t)img_bytes};
    const cuuint32_t box[4] = {32, (cuuint32_t)W, (cuuint32_t)W, 1};
    const cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&maps.m4, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, buf, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode 4d failed %d\n", (int)r); return 1; }
  }
  const int box_rows = W * W, box_bytes = box_rows * 128;
  const int nbox = (int)((size_t)nimg * img_bytes / box_bytes);
  {
    const cuuint64_t dims[2] = {32, (cuuint64_t)nbox * box_rows};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    const cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&maps.m2, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, buf, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("encode 2d failed %d\n", (int)r); return 1; }
  }
  const int grid = p.multiProcessorCount * per_sm;
  const size_t smem = (size_t)stages * ((box_bytes + 1023) / 1024 * 1024) + 1024;
  CK(cudaFuncSetAttribute(tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int iters = 600;
  const char* names[3] = {"4-D strided box", "2-D dense box  ", "linear bulk    "};
  for (int mode = 0; mode < 3; ++mode)
    for (int rep = 0; rep < 2; ++rep) {
      const int n = mode == 0 ? nimg : nbox;
      CK(cudaEventRecord(e0));
      tma_kernel<<<grid, 32, smem>>>(maps, buf, mode, n, box_bytes, stages, iters, sink);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      const double bytes = (double)grid * iters * box_bytes;
      printf("%s W=%d stride=%d box=%d B stages=%d ctas/sm=%d : %.3f ms  %.2f TB/s  %.2f us/box/SM-slot\n", names[mode], W, stride,
             box_bytes, stages, per_sm, ms, bytes / ms * 1e-9, ms * 1e3 / iters);
    }
  return 0;
}
