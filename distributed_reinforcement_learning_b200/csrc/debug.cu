// debug.cu -- drl_debug_gemm: runs ONE plain GEMM  C[M,N] = A * B  on either contraction core
// (FP32-FFMA gather-GEMM or wgmma 3xTF32) with every operand-major combination the layers use,
// so the shared-memory layouts / wgmma descriptors can be validated in isolation against NumPy.
#include <vector>

#include "gemm_simt.cuh"
#include "gemm_umma.cuh"
#include "gemm_umma16.cuh"
#include "kernels.h"
#include "loaders.cuh"

namespace drl {

// cores 5 / 6: 16-bit split operands (bf16 / fp16), B gathered by the producers; cores 7 / 8: the same with B fetched
// from a pre-tiled K-major image by the loader warp (kchunk rounded to 64)
template <class F, class AL, class BL, class EP>
static int run_fmt16(bool pretiled, int bn, cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                     int nz, int kchunk) {
  if (!pretiled) {
    if (!BL::kContigK && bn < 64) { set_error("debug_gemm: MN-major 16-bit B tiles need bn >= 64"); return DRL_ERR_INVALID; }
    switch (bn) {
      case 32: if constexpr (BL::kContigK) return launch_gemm_umma16<Umma16Cfg<32, 2, 1, 4, 0, F, F>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk); else break;
      case 64: return launch_gemm_umma16<Umma16Cfg<64, 2, 1, 4, 0, F, F>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
      case 128: return launch_gemm_umma16<Umma16Cfg<128, 3, 1, 8, 0, F, F>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
      case 256: return launch_gemm_umma16<Umma16Cfg<256, 2, 1, 4, 0, F, F>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
    }
    set_error("debug_gemm: bn must be 32 (K-major B), 64, 128 or 256");
    return DRL_ERR_INVALID;
  }
  uint8_t* img = nullptr;
  int rc = DRL_ERR_INVALID;
  auto with_image = [&](auto bn_tag) -> int {
    constexpr int BN = decltype(bn_tag)::value;
    DRL_CUDA_CHECK(cudaMalloc(&img, weight_image16_bytes<BN>(N, K) + 1024));
    DRL_TRY((launch_retile_b16<BN, F>(s, bl, N, K, img)));
    PretiledB<BL> blp{img, cdiv(K, 64)};
    using Cfg = Umma16Cfg<BN, (BN == 256 ? 2 : 3), 1, (BN == 128 ? 8 : 4), (BN == 256 ? 0 : 1), F, F>;
    return launch_gemm_umma16<Cfg>(s, al, blp, ep, M, N, K, nz, kchunk, kchunk);
  };
  switch (bn) {
    case 32: rc = with_image(std::integral_constant<int, 32>{}); break;
    case 64: rc = with_image(std::integral_constant<int, 64>{}); break;
    case 128: rc = with_image(std::integral_constant<int, 128>{}); break;
    case 256: rc = with_image(std::integral_constant<int, 256>{}); break;
    default: set_error("debug_gemm: bn must be 32, 64, 128 or 256");
  }
  cudaStreamSynchronize(s);
  if (img) cudaFree(img);
  return rc;
}
template <class AL, class BL, class EP>
static int run_one16(int core, int bn, cudaStream_t s, const AL& al, const BL& bl, const EP& ep, int M, int N, int K,
                     int nz, int kchunk) {
  const bool pre = core >= 7;
  if (pre) kchunk = (kchunk + 63) / 64 * 64;
  if (core == 5 || core == 7) return run_fmt16<umma16::BF16>(pre, bn, s, al, bl, ep, M, N, K, (K + kchunk - 1) / kchunk, kchunk);
  if (core == 6 || core == 8) return run_fmt16<umma16::F16>(pre, bn, s, al, bl, ep, M, N, K, (K + kchunk - 1) / kchunk, kchunk);
  set_error("debug_gemm: unknown core %d", core);
  return DRL_ERR_INVALID;
}

template <class AL, class BL>
static int run_one(int core, int bn, cudaStream_t s, const AL& al, const BL& bl, float* C, int M, int N, int K,
                   int splits) {
  int kchunk = (K + splits - 1) / splits;
  kchunk = (kchunk + 31) / 32 * 32;
  const int nz = (K + kchunk - 1) / kchunk;
  EpRaw<true> ep{C, N, (size_t)(M + 1) * N, 1.0f, M, N};     // slab z: [M+1, N], row M = column sums of B
  if (core == 1) return launch_gemm_simt<CfgMid>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
  if (core >= 5) return run_one16(core, bn, s, al, bl, ep, M, N, K, nz, kchunk);
  switch (bn) {
    case 32: return launch_gemm_umma<UmmaCfg<32, 2, 1>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
    case 64: return launch_gemm_umma<UmmaCfg<64, 2, 1>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
    case 128: return launch_gemm_umma<UmmaCfg<128, 3, 1, 8>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
    case 256: return launch_gemm_umma<UmmaCfg<256, 2, 1, 4>>(s, al, bl, ep, M, N, K, nz, kchunk, kchunk);
    default: set_error("debug_gemm: bn must be 32, 64, 128 or 256"); return DRL_ERR_INVALID;
  }
}

}  // namespace drl

using namespace drl;

// core: 1 = FFMA, 2 = wgmma 3xTF32, 5-8 = wgmma 16-bit split (see run_one16).  a_kmajor: A given as [M,K] row-major (1) or as [K,M] row-major (0).
// b_kmajor: B given as [N,K] row-major (1) or [K,N] row-major (0).  C out: [splits][(M+1), N] host floats
// (row M of each slab = column sums of B over that split's K range when B is N-major, else untouched).
extern "C" int drl_debug_gemm(int32_t core, int32_t bn, int32_t a_kmajor, int32_t b_kmajor, int32_t M, int32_t N,
                              int32_t K, int32_t splits, const float* A, const float* B, float* C) {
  if (!A || !B || !C || M < 1 || N < 1 || K < 1 || splits < 1) { set_error("debug_gemm: bad argument"); return DRL_ERR_INVALID; }
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  float *dA = nullptr, *dB = nullptr, *dC = nullptr;
  const size_t nA = (size_t)M * K, nB = (size_t)N * K, nC = (size_t)splits * (M + 1) * N;
  DRL_CUDA_CHECK(cudaMalloc(&dA, nA * 4 + 64));
  DRL_CUDA_CHECK(cudaMalloc(&dB, nB * 4 + 64));
  DRL_CUDA_CHECK(cudaMalloc(&dC, nC * 4 + 64));
  DRL_CUDA_CHECK(cudaMemcpy(dA, A, nA * 4, cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemcpy(dB, B, nB * 4, cudaMemcpyHostToDevice));
  DRL_CUDA_CHECK(cudaMemset(dC, 0, nC * 4));
  int rc;
  if (a_kmajor && b_kmajor) rc = run_one(core, bn, 0, PlainA{dA, K, 0}, PlainBT{dB, K, 0}, dC, M, N, K, splits);
  else if (a_kmajor && !b_kmajor) rc = run_one(core, bn, 0, PlainA{dA, K, 0}, PlainB{dB, N, 0}, dC, M, N, K, splits);
  else if (!a_kmajor && b_kmajor) rc = run_one(core, bn, 0, PlainAT{dA, M, 0}, PlainBT{dB, K, 0}, dC, M, N, K, splits);
  else rc = run_one(core, bn, 0, PlainAT{dA, M, 0}, PlainB{dB, N, 0}, dC, M, N, K, splits);
  cudaError_t e = cudaDeviceSynchronize();
  if (rc == DRL_OK && e != cudaSuccess) { set_error("debug_gemm kernel failed: %s", cudaGetErrorString(e)); rc = DRL_ERR_CUDA; }
  if (rc == DRL_OK) {
    e = cudaMemcpy(C, dC, nC * 4, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error("debug_gemm copy failed: %s", cudaGetErrorString(e)); rc = DRL_ERR_CUDA; }
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dC);
  return rc;
}
