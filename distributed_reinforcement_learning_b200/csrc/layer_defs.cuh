// layer_defs.cuh -- loader / tile-configuration instantiations, launch macros, split-K plans and the conv trunk's
// forward and backward shared by the IMPALA actor-critic (layers.cu), the Ape-X / A3C network (apex.cu) and the R2D2
// network (r2d2.cu): all run the same attention_CNN (model/impala_actor_critic.py:5-10 == model/apex_value.py:4-9)
// through the same gather-GEMM kernels.
#pragma once
#include <algorithm>

#include "gemm_simt.cuh"
#include "gemm_umma.cuh"
#include "gemm_umma16.cuh"
#include "conv1_tma.cuh"
#include "gemm_bulk16.cuh"
#include "gemm_umma_persist.cuh"
#include "kernels.h"
#include "loaders.cuh"
#include "trunk_images.cuh"

namespace drl {

// ------------------------------------------------------------------------------------------
// Loader / epilogue instantiations for the three convolutions
// ------------------------------------------------------------------------------------------
using Conv1A = ConvFwdA<uint8_t, 84, 84, 4, 20, 20, 8, 4, true>;
using Conv2A = ConvFwdA<float, 20, 20, 32, 9, 9, 4, 2, false>;
using Conv3A = ConvFwdA<float, 9, 9, 64, 7, 7, 3, 1, false>;
using Conv1WA = ConvWgradA<uint8_t, 84, 84, 4, 20, 20, 8, 4, true>;
using Conv2WA = ConvWgradA<float, 20, 20, 32, 9, 9, 4, 2, false>;
using Conv3WA = ConvWgradA<float, 9, 9, 64, 7, 7, 3, 1, false>;
using Conv3DA = ConvDgradA<7, 7, 64, 1, 3, 3, 9, 9>;
using Conv3DB = ConvDgradB<64, 64, 1, 3, 3>;
using Conv3DE = EpConvDx<9, 9, 64, 1, 9, 9>;
using Conv2DA = ConvDgradA<9, 9, 64, 2, 4, 4, 10, 10>;
using Conv2DB = ConvDgradB<32, 64, 2, 4, 4>;
using Conv2DE = EpConvDx<20, 20, 32, 2, 10, 10>;
using Conv2DBm = ConvDgradBMerged<32, 64, 2, 4, 4>;     // math mode 5: the four parity classes as one GEMM, N = 128
using Conv2DEm = EpConvDxMerged<20, 20, 32, 2, 10, 10>;
// math mode 5: the same A operands read from the 16-bit planes of a1 / a2 / da3 / da2 (cp.async, no fp32 gather)
using Conv2AP = PlaneA<Conv2A>;
using Conv3AP = PlaneA<Conv3A>;
using Conv3DAP = PlaneA<Conv3DA>;
using Conv2DAP = PlaneA<Conv2DA>;

// Every tensor-core configuration has two consumer warpgroups (256 threads) whose wgmma accumulators hold BN / 2 fp32
// registers per thread, next to the producer warps, in one CTA per SM unless MINB says otherwise: BN = 256 (128
// accumulator registers) leaves room for 4 producer warps and no loader warp within the 65,536 registers of an H100 SM.
using U32 = UmmaCfg<32, 2, 1>;   // 24 KB / stage (A exact: conv1 only)
using U64 = UmmaCfg<64, 2, 1>;   // 48 KB / stage
using U128 = UmmaCfg<128, 3, 1, 8>;   // 64 KB / stage, 8 producer warps
using U256 = UmmaCfg<256, 2, 1, 4>;   // 96 KB / stage, 4 producer warps
// the same for GEMMs whose B operand is a pre-tiled weight image (B-loader warp where the registers allow it)
using U64L = UmmaCfg<64, 2, 1, 4, 1>;
using U128L = UmmaCfg<128, 3, 1, 8, 1>;
using U256L = U256;                    // (no loader warp: the same configuration as U256)

// math mode 5: 16-bit split operands (gemm_umma16.cuh).  One format per GEMM (f16 x bf16 traps).  bf16 keeps fp32's
// exponent range (gradients span many decades); fp16 has three more mantissa bits but underflows gradually below ~1e-4
// and saturates at 65504 -- conv1 (conv1_tma.cuh) uses it because one operand is EXACT in it (the uint8 frames) and the
// other is an O(0.1) weight.
using Fmt16 = umma16::BF16;     // every GEMM whose operands are fp32 activations / gradients / weights
// Two CTAs per SM (MINB = 2, 106 KB of shared memory each): one CTA's pipeline fill and epilogue overlap the other's main
// loop.  512 threads x 64 registers, split by role: 8 producer warps keep PREG registers and issue the weight image's bulk
// copy themselves, the consumer warpgroups take the rest.  Fed from planes (PlaneA), the producers only compute addresses
// and issue cp.async; the register prefetch ring of the fp32 gather path does not apply.
using X64L2 = Umma16Cfg<64, 2, 2, 8, 0, Fmt16, Fmt16, 0, false, 56>;  // conv2 / conv3 fwd: 48 KB per K = 64 stage; producers
                                                                     // 56 (a prefetch ring of 2 sub-tiles), consumers 72
using X64W8x2 = Umma16Cfg<64, 2, 1, 8, 0, Fmt16, Fmt16>;     // conv2 / conv3 weight gradients (both operands gathered)
using XH = Umma16Cfg<64, 4, 1, 8, 0, Fmt16, Fmt16>;          // head layers (K = 256 = all four stages in flight)
// bulk-fed LSTM weight gradient (gemm_bulk16.cuh): both operands are pre-tiled images, no producer warps
using BK256 = Bulk16Cfg<256, 2>;       // 96 KB per stage (A 32 KB + B 64 KB), 2 stages
using X256L = Umma16Cfg<256, 2, 1, 4, 0, Fmt16, Fmt16>;      // lstm fwd: 96 KB per stage
using X128D = Umma16Cfg<128, 3, 1, 8, 1, Fmt16, Fmt16>;      // lstm data gradient: 64 KB per stage
// conv data gradients (pre-tiled B, one K tile of 64 co per filter tap, A copied from the da3 / da2 planes): per-tap
// partial sums added in tap order, the rounding of the dCol GEMM + col2im of math modes 2 and 3.  Two CTAs per SM as
// X64L2; the second register set (64 per consumer thread) leaves the producers 48 registers, which the plane copies'
// addresses fit.  conv3: K = 9 taps x 64 co, N = 64 ci.  conv2: K = 4 taps x 64 co, N = 4 parity classes x 32 ci, as two
// N tiles of (py, px = 0..1) x 32 ci (each N tile copies the dY taps itself: ~59 MB more L2 reads at B = 32, T = 20).
// (conv3's data gradient with the fp32 register gather measured slower at two CTAs per SM than at one, 0.070 -> 0.072
// ms; fed from its plane it measured faster, 0.057 -> 0.052 ms, on an H100 SXM at 700 W.)
using X64T2 = Umma16Cfg<64, 2, 2, 8, 0, Fmt16, Fmt16, 0, true, 48>;

// math mode 3 (experimental): the persistent, fully warp-specialised variant of each tensor-core configuration
template <class U> struct PersistOf;
template <> struct PersistOf<U32> { using type = UmmaPCfg<32, 5, 8>; };
template <> struct PersistOf<U64> { using type = UmmaPCfg<64, 4, 8>; };
template <> struct PersistOf<U128> { using type = UmmaPCfg<128, 3, 8>; };
template <> struct PersistOf<U256> { using type = UmmaPCfg<256, 2, 4>; };
template <> struct PersistOf<U64L> { using type = UmmaPCfg<64, 4, 8>; };
template <> struct PersistOf<U128L> { using type = UmmaPCfg<128, 3, 8>; };


// name the launch for the per-kernel profile, run it on the selected core, count it
#define GEMM(name, SCfg, UCfg, ...)                          \
  do {                                                       \
    prof_mark(s, name);                                      \
    if (mode == 3) {                                         \
      DRL_TRY((launch_gemm_umma_persist<typename PersistOf<UCfg>::type>(s, __VA_ARGS__))); \
    } else if (mode == 2 || mode == 5) {                     \
      DRL_TRY((launch_gemm_umma<UCfg>(s, __VA_ARGS__)));     \
    } else {                                                 \
      DRL_TRY((launch_gemm_simt<SCfg>(s, __VA_ARGS__)));     \
    }                                                        \
    ++n;                                                     \
  } while (0)
// a GEMM on the 16-bit split core (math mode 5)
#define GEMM16(name, XCfg, ...)                              \
  do {                                                       \
    prof_mark(s, name);                                      \
    DRL_TRY((launch_gemm_umma16<XCfg>(s, __VA_ARGS__)));     \
    ++n;                                                     \
  } while (0)
// same, for GEMMs whose B operand is a weight matrix: the tensor-core cores read its pre-tiled image (blp)
#define GEMM_W(name, SCfg, UCfg, al, bl, blp, ...)            \
  do {                                                       \
    prof_mark(s, name);                                      \
    if (mode == 3) {                                         \
      DRL_TRY((launch_gemm_umma_persist<typename PersistOf<UCfg>::type>(s, al, blp, __VA_ARGS__))); \
    } else if (mode == 2) {                                  \
      DRL_TRY((launch_gemm_umma<UCfg>(s, al, blp, __VA_ARGS__))); \
    } else {                                                 \
      DRL_TRY((launch_gemm_simt<SCfg>(s, al, bl, __VA_ARGS__))); \
    }                                                        \
    ++n;                                                     \
  } while (0)
#define GEMM_FFMA(name, SCfg, ...)                           \
  do {                                                       \
    prof_mark(s, name);                                      \
    DRL_TRY((launch_gemm_simt<SCfg>(s, __VA_ARGS__)));       \
    ++n;                                                     \
  } while (0)
// the small dense layers of the heads: in-CTA split-K (KS groups work on the K tiles of one output tile concurrently)
#define GEMM_FFMA_KS(name, SCfg, KS, ...)                      \
  do {                                                       \
    prof_mark(s, name);                                      \
    DRL_TRY((launch_gemm_simt<SCfg, KS>(s, __VA_ARGS__)));   \
    ++n;                                                     \
  } while (0)
#define KERNEL(name, call, cnt)                              \
  do {                                                       \
    prof_mark(s, name);                                      \
    DRL_TRY(call);                                           \
    n += (cnt);                                              \
  } while (0)

// split-K plan: about `waves` waves of CTAs on the 132 SMs of an H100
struct SplitPlan { int splits, kchunk; };
static SplitPlan plan_split(int K, int tiles_mn, int bk, int waves) {
  int target = (waves * 132 + tiles_mn - 1) / tiles_mn;
  if (target < 1) target = 1;
  int kchunk = (K + target - 1) / target;
  kchunk = (kchunk + bk - 1) / bk * bk;
  if (kchunk < bk) kchunk = bk;
  SplitPlan p;
  p.kchunk = kchunk;
  p.splits = (K + kchunk - 1) / kchunk;
  return p;
}
// the conv weight-gradient plans (mode 1: FFMA tiles, 2 waves; mode 2: 128-row UMMA tiles, 2 CTAs/SM)
static SplitPlan plan_conv1_wgrad(int Mb, int mode) {
  return mode >= 2 ? plan_split(Mb * 400, 2, 32, 2) : plan_split(Mb * 400, cdiv(256, CfgWg1::BM), 16, 2);
}
// conv1 weight gradient with single-channel frames (R2D2) is a [64 x 32] output with K = Mb*400: half of a 128-row MMA
// tile would be padding and the producers, not the tensor pipe, set the pace on the 128-row tensor-core core.  A 64 x 32
// FFMA tile with the reduction split over ~4 CTAs per SM fits the shape in both math modes.
using CfgWgC1 = TileCfg<64, 32, 16, 4, 4>;
static SplitPlan plan_conv1_wgrad_c1(int Mb) { return plan_split(Mb * 400, 1, 16, 4); }
static SplitPlan plan_conv2_wgrad(int Mb, int mode) {
  if (mode == 5) return plan_split(Mb * 81, 4, 64, 2);
  return mode >= 2 ? plan_split(Mb * 81, 4, 32, 2) : plan_split(Mb * 81, cdiv(512, CfgBig::BM), 16, 2);
}
static SplitPlan plan_conv3_wgrad(int Mb, int mode) {
  if (mode == 5) return plan_split(Mb * 49, 5, 64, 2);
  return mode >= 2 ? plan_split(Mb * 49, 5, 32, 2) : plan_split(Mb * 49, cdiv(576, CfgBig::BM), 16, 2);
}

// The conv1 / conv2 / conv3 forward of every network's trunk over B sequences of S frames of C channels (rows m = t*B + b;
// S = 1: the caller's row order) on stream s, with the learner's kernels and configurations for math mode `mode` (1: FP32
// FFMA; 2 and 3: wgmma 3xTF32 with the conv2 / conv3 weight images of conv_images_tf32).  When images_ready is not null,
// conv2 waits for it (the images are built on another stream).  `tgt` only names the launches for the per-kernel
// profile; adds the launches to *launches.  Defined here so that each learner (layers.cu, apex.cu, r2d2.cu) instantiates
// the kernels it launches; the Ape-X / A3C and R2D2 policy engines reach it through policy_conv_forward_tf32 (r2d2.cu).
template <int C>
int conv_forward_tf32(cudaStream_t s, const TrunkLayout& pl, const float* P, const uint8_t* img_conv2,
                      const uint8_t* img_conv3, const uint8_t* frames, int B, int S, float* a1, float* a2, float* a3,
                      int mode, bool tgt, cudaEvent_t images_ready, int* launches) {
  const int M = B * S;
  const RowMap map{B, S};
  int n = 0;
  {
    ConvFwdA<uint8_t, 84, 84, C, 20, 20, 8, 4, true> al{frames, map};
    PlainB bl{P + pl.conv1_w, 32, 0};
    EpConv1 ep{a1, 32, P + pl.conv1_b};
    GEMM(tgt ? "target_conv1_fwd" : "conv1_fwd", CfgN32, U32, al, bl, ep, M * 400, 32, 64 * C, 1, 64 * C, 0);
  }
  if (images_ready) DRL_CUDA_CHECK(cudaStreamWaitEvent(s, images_ready, 0));
  {
    Conv2A al{a1, map};
    PlainB bl{P + pl.conv2_w, 64, 0};
    PretiledB<PlainB> blp{img_conv2, 512 / 32};
    EpBiasAct<true, true> ep{a2, 64, 0, P + pl.conv2_b, 0, 1.0f};
    GEMM_W(tgt ? "target_conv2_fwd" : "conv2_fwd", CfgBig, U64L, al, bl, blp, ep, M * 81, 64, 512, 1, 512, 0);
  }
  {
    Conv3A al{a2, map};
    PlainB bl{P + pl.conv3_w, 64, 0};
    PretiledB<PlainB> blp{img_conv3, 576 / 32};
    EpBiasAct<true, true> ep{a3, 64, 0, P + pl.conv3_b, 0, 1.0f};
    GEMM_W(tgt ? "target_conv3_fwd" : "conv3_fwd", CfgBig, U64L, al, bl, blp, ep, M * 49, 64, 576, 1, 576, 0);
  }
  *launches += n;
  return DRL_OK;
}

// Fork/join helpers: kernels that are off the critical path (the action-embedding table in the forward, every
// weight gradient except conv1's in the backward) run on the side stream so they fill SMs the critical
// dgrad chain leaves idle.  Inside CUDA-graph capture the event record/wait pairs become graph edges.
static inline int fork_to_side(const Streams& st, int i) {
  if (!st.par) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventRecord(st.ev[i], st.main));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(st.side, st.ev[i], 0));
  return DRL_OK;
}
// main -> side2 edge (ev2[i]); side2 -> other stream edge
static inline int fork_to_side2(const Streams& st, int i) {
  if (!st.par || !st.side2) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventRecord(st.ev2[i], st.main));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(st.side2, st.ev2[i], 0));
  return DRL_OK;
}
static inline int join_side2_into(const Streams& st, int i, cudaStream_t into) {
  if (!st.par || !st.side2) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventRecord(st.ev2[i], st.side2));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(into, st.ev2[i], 0));
  return DRL_OK;
}
static inline int join_from_side(const Streams& st, int i) {
  if (!st.par) return DRL_OK;
  DRL_CUDA_CHECK(cudaEventRecord(st.ev[i], st.side));
  DRL_CUDA_CHECK(cudaStreamWaitEvent(st.main, st.ev[i], 0));
  return DRL_OK;
}

// The conv trunk backward in math modes 1 to 3 over Mb rows (row order `map`, the forward's), from "da3 ready on main,
// side forked at ev[4]" to the conv1 weight-gradient reduce: the conv3 / conv2 weight gradients on the side stream, the
// data gradients on main (modes 2 and 3: the dCol GEMM with the img[5] / img[6] images of conv_dcol_images_tf32, then
// col2im; mode 1: the FFMA gather), then conv1's weight gradient on main.  The caller joins side back at ev[6].  Adds
// the launches to *launches; a template like conv_forward_tf32.
template <int C>
int conv_backward_tf32(const Streams& st, const TrunkLayout& pl, const float* P, const WeightImages& wi, float* G,
                       const uint8_t* frames, RowMap map, int Mb, const TrunkActs& act, const TrunkBwd& bw, int mode,
                       int* launches) {
  cudaStream_t s = st.par ? st.side : st.main;
  int n = 0;
  {
    const SplitPlan sp = plan_conv3_wgrad(Mb, mode);
    const size_t slab = 577 * 64;
    Conv3WA al{act.a2, map};
    PlainB bl{bw.da3, 64, 0};
    EpRaw<true> ep{bw.wg_part, 64, slab, 1.0f, 576, 64};
    GEMM("conv3_wgrad", CfgBig, U64, al, bl, ep, 576, 64, Mb * 49, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv3_wgrad_reduce", splitk_reduce(s, bw.wg_part, slab, sp.splits, G + pl.conv3_w, slab), 1);
  }
  s = st.main;
  if (mode >= 2) {
    // "dCol" form: one plain GEMM with K = 64 output channels (instead of gathering every dY value 9 times
    // through the producers), then a gather of <= 9 taps per input pixel with the ReLU mask.  K = 64 (two K tiles) and
    // 128 x 256 outputs per tile: epilogue-dominated, so the persistent kernel whose dedicated epilogue warps wins here
    // while the producers gather the next tile.
    PlainA al{bw.da3, 64, 0};
    EpRaw<false> ep{bw.dcol, 576, 0, 1.0f, 0, 576};
    prof_mark(s, "conv3_dgrad");
    PretiledB<PlainBT> blp{wi.img[5], 2};   // B(k = co, n = (ky,kx,ci)) = W[n*64 + co]
    DRL_TRY((launch_gemm_umma_persist<PersistOf<U256>::type>(s, al, blp, ep, Mb * 49, 576, 64, 1, 64, 0)));
    prof_mark(s, "conv3_col2im");
    DRL_TRY(col2im_conv3(s, bw.dcol, act.a2, bw.da2, Mb));
    n += 2;
  } else {
    Conv3DA al{bw.da3};
    Conv3DB bl{P + pl.conv3_w};
    Conv3DE ep{bw.da2, act.a2};
    GEMM_FFMA("conv3_dgrad", CfgBig, al, bl, ep, Mb * 81, 64, 576, 1, 576, 0);
  }
  DRL_TRY(fork_to_side(st, 5));
  s = st.par ? st.side : st.main;
  {
    const SplitPlan sp = plan_conv2_wgrad(Mb, mode);
    const size_t slab = 513 * 64;
    Conv2WA al{act.a1, map};
    PlainB bl{bw.da2, 64, 0};
    EpRaw<true> ep{bw.wg_part, 64, slab, 1.0f, 512, 64};
    GEMM("conv2_wgrad", CfgBig, U64, al, bl, ep, 512, 64, Mb * 81, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv2_wgrad_reduce", splitk_reduce(s, bw.wg_part, slab, sp.splits, G + pl.conv2_w, slab), 1);
  }
  s = st.main;
  if (mode >= 2) {
    PlainA al{bw.da2, 64, 0};
    EpRaw<false> ep{bw.dcol, 512, 0, 1.0f, 0, 512};
    prof_mark(s, "conv2_dgrad");                      // persistent kernel: 0.079 vs 0.091 ms
    PretiledB<PlainBT> blp{wi.img[6], 2};
    DRL_TRY((launch_gemm_umma_persist<PersistOf<U256>::type>(s, al, blp, ep, Mb * 81, 512, 64, 1, 64, 0)));
    prof_mark(s, "conv2_col2im");
    DRL_TRY(col2im_conv2(s, bw.dcol, act.a1, bw.da1, Mb));
    n += 2;
  } else {
    Conv2DA al{bw.da2};
    Conv2DB bl{P + pl.conv2_w};
    Conv2DE ep{bw.da1, act.a1};
    GEMM_FFMA("conv2_dgrad", CfgN32, al, bl, ep, Mb * 100, 32, 256, 4, 256, 0);
  }
  // conv1 (input is data: weight gradient only), own partial buffer: runs beside the side stream
  ConvWgradA<uint8_t, 84, 84, C, 20, 20, 8, 4, true> al{frames, map};
  PlainB bl{bw.da1, 32, 0};
  const size_t slab = (64 * C + 1) * 32;
  EpRaw<true> ep{bw.wg_part2, 32, slab, 1.0f / 255.0f, 64 * C, 32};
  if constexpr (C == 1) {
    const SplitPlan sp = plan_conv1_wgrad_c1(Mb);
    GEMM_FFMA("conv1_wgrad", CfgWgC1, al, bl, ep, 64, 32, Mb * 400, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv1_wgrad_reduce", splitk_reduce(s, bw.wg_part2, slab, sp.splits, G + pl.conv1_w, slab), 1);
  } else {
    const SplitPlan sp = plan_conv1_wgrad(Mb, mode);
    GEMM("conv1_wgrad", CfgWg1, U32, al, bl, ep, 256, 32, Mb * 400, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv1_wgrad_reduce", splitk_reduce(s, bw.wg_part2, slab, sp.splits, G + pl.conv1_w, slab), 1);
  }
  *launches += n;
  return DRL_OK;
}

}  // namespace drl
