// p2p_bw.cu -- NVLink peer-memory bandwidth seen by a kernel on GPU 0 that reads / writes GPU 1's memory with
// 128-bit accesses (the access pattern of csrc/peer.cu), for a slice-sized (8 MB) and a large (128 MB) buffer.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o p2p_bw p2p_bw.cu     Usage: ./p2p_bw
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

template <int U>
__global__ void rd(const float4* __restrict__ src, float4* __restrict__ dst_local, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float4 acc = make_float4(0, 0, 0, 0);
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += U * stride) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { size_t i = i0 + u * stride; v[u] = i < n ? __ldcg(src + i) : make_float4(0, 0, 0, 0); }
#pragma unroll
    for (int u = 0; u < U; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
  }
  if (acc.x == 1234.5f) dst_local[0] = acc;
}
__global__ void wr(float4* __restrict__ dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = make_float4(1, 2, 3, 4);
}
__global__ void rdwr(const float4* __restrict__ src, float4* __restrict__ dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = __ldcg(src + i);
}

int main() {
  int nd = 0; CK(cudaGetDeviceCount(&nd));
  if (nd < 2) { printf("needs 2 GPUs\n"); return 0; }
  int can = 0; CK(cudaDeviceCanAccessPeer(&can, 0, 1)); printf("canAccessPeer(0,1) = %d\n", can);
  CK(cudaSetDevice(0)); CK(cudaDeviceEnablePeerAccess(1, 0));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  for (size_t mb : {8, 128}) {
    const size_t bytes = mb << 20, n = bytes / 16;
    float4 *remote, *remote2, *local;
    CK(cudaSetDevice(1)); CK(cudaMalloc(&remote, bytes)); CK(cudaMalloc(&remote2, bytes)); CK(cudaMemset(remote, 0, bytes));
    CK(cudaSetDevice(0)); CK(cudaMalloc(&local, bytes)); CK(cudaMemset(local, 0, bytes));
    CK(cudaDeviceSynchronize());
    for (int grid : {296, 592, 1184}) {
      float ms;
      for (int rep = 0; rep < 2; ++rep) { CK(cudaEventRecord(e0)); rd<4><<<grid, 256>>>(remote, local, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); }
      printf("%4zu MB grid %4d  remote read  U=4: %7.1f us  %6.1f GB/s\n", mb, grid, ms * 1e3, bytes / ms * 1e-6);
      for (int rep = 0; rep < 2; ++rep) { CK(cudaEventRecord(e0)); rd<1><<<grid, 256>>>(remote, local, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); }
      printf("%4zu MB grid %4d  remote read  U=1: %7.1f us  %6.1f GB/s\n", mb, grid, ms * 1e3, bytes / ms * 1e-6);
      for (int rep = 0; rep < 2; ++rep) { CK(cudaEventRecord(e0)); wr<<<grid, 256>>>(remote2, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); }
      printf("%4zu MB grid %4d  remote write     : %7.1f us  %6.1f GB/s\n", mb, grid, ms * 1e3, bytes / ms * 1e-6);
      for (int rep = 0; rep < 2; ++rep) { CK(cudaEventRecord(e0)); rdwr<<<grid, 256>>>(remote, remote2, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); }
      printf("%4zu MB grid %4d  remote rd+wr     : %7.1f us  %6.1f GB/s each way\n", mb, grid, ms * 1e3, bytes / ms * 1e-6);
    }
    float ms;
    for (int rep = 0; rep < 2; ++rep) { CK(cudaEventRecord(e0)); CK(cudaMemcpyPeerAsync(local, 0, remote, 1, bytes)); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); CK(cudaEventElapsedTime(&ms, e0, e1)); }
    printf("%4zu MB cudaMemcpyPeer          : %7.1f us  %6.1f GB/s\n", mb, ms * 1e3, bytes / ms * 1e-6);
  }
  return 0;
}
