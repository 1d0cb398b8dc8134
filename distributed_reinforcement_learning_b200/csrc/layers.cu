// layers.cu -- forward and backward of the IMPALA actor-critic (model/impala_actor_critic.py:33-42)
// over M = B*T independent rows (the LSTM is a single step from fed state, :18-25 / :73-82, so
// time is embarrassingly parallel; only T distinct forwards exist, SURVEY.md section 0.3).
// Every dense contraction is one launch of a gather-GEMM: the FP32-FFMA core (gemm_simt.cuh, math
// mode 1) or the wgmma 3xTF32 tensor-core core (gemm_umma.cuh, math mode 2) -- same loaders and
// epilogues.  Outside math mode 5 the small head layers (M x 256 x 256) use the FFMA core.
#include "layer_defs.cuh"
#include "r2d2_cluster.cuh"

namespace drl {

// ------------------------------------------------------------------------------------------
// Recurrent mode (Recurrence, kernels.h; DESIGN.md section 21): the LSTM of each trajectory runs through its T steps
// on the cluster kernels of r2d2_cluster.cuh at L = 256, RESTART variant: step 0 and every step after a done start from
// the state the actor recorded for it, every other step from the previous step's output.  The BPTT walks the T - 2
// steps that receive loss gradient (the time-major prefix of Mb = B (T - 2) rows) and carries nothing across a done.
// ------------------------------------------------------------------------------------------
using ImpClu = R2Clu<Geo::L>;

__global__ void __launch_bounds__(ImpClu::T, 1) impala_lstm_fwd_cluster_kernel(
    const float* __restrict__ zx, const float* __restrict__ bias, const float* __restrict__ Wh,
    const float* __restrict__ h0, const float* __restrict__ c0, const uint8_t* __restrict__ done,
    float* __restrict__ gates, float* __restrict__ tc, float* __restrict__ hout, float* __restrict__ hin,
    float* __restrict__ cin, float* __restrict__ c_last, int B, int T) {
  lstm_fwd_cluster_body<Geo::L, true>(zx, bias, Wh, h0, c0, done, gates, tc, hout, hin, cin, c_last, B, T);
}

__global__ void __launch_bounds__(ImpClu::T, 1) impala_lstm_bwd_cluster_kernel(
    const float* __restrict__ dh_part, size_t part_stride, const float* __restrict__ gates,
    const float* __restrict__ tc, const float* __restrict__ cin, const float* __restrict__ Wh,
    const uint8_t* __restrict__ done, float* __restrict__ dz, int B, int T) {
  lstm_bwd_cluster_body<Geo::L, true>(dh_part, part_stride, gates, tc, cin, Wh, done, dz, B, T - 2, T);
}

int impala_recurrence_setup(Recurrence* rec) {
  return lstm_cluster_setup<Geo::L>(impala_lstm_fwd_cluster_kernel, impala_lstm_bwd_cluster_kernel, &rec->clusters_fwd,
                                    &rec->clusters_bwd);
}

// one cluster per R = 8 trajectories, up to what the device places at once
static int recurrence_grid(int B, int max_clusters) { return std::min(cdiv(B, ImpClu::R), max_clusters) * ImpClu::CL; }

void FlatLayout::set(int n, const int64_t* sizes, int64_t* const* named) {
  num_tensors = n;
  int64_t po = 0, pk = 0;
  for (int i = 0; i < n; ++i) {
    count[i] = sizes[i];
    packed_off[i] = pk;
    padded_off[i] = po;
    pk += sizes[i];
    po += sizes[i];
    if (i & 1) po = (po + 3) / 4 * 4;   // pad after each bias (all kernel sizes are multiples of 4)
    *named[i] = padded_off[i];
  }
  packed_total = pk;
  padded_total = (po + 3) / 4 * 4;
}

void ParamLayout::init(int num_action) {
  A = num_action;
  const int64_t sizes[] = {
      8 * 8 * 4 * 32, 32, 4 * 4 * 32 * 64, 64, 3 * 3 * 64 * 64, 64,
      (int64_t)A * 256, 256, 256 * 256, 256,
      (int64_t)Geo::XK * Geo::G4, Geo::G4,
      256 * 256, 256, 256 * 256, 256, 256 * (int64_t)A, A,
      256 * 256, 256, 256 * 256, 256, 256, 1};
  int64_t* const named[] = {&conv1_w, &conv1_b, &conv2_w, &conv2_b, &conv3_w, &conv3_b, &emb1_w, &emb1_b,
                            &emb2_w, &emb2_b, &lstm_w, &lstm_b, &actor1_w, &actor1_b, &actor2_w, &actor2_b,
                            &actor3_w, &actor3_b, &critic1_w, &critic1_b, &critic2_w, &critic2_b, &critic3_w,
                            &critic3_b};
  set(sizes, named);
}

static int g_fwd_launches = 0, g_bwd_launches = 0;
int forward_launch_count() { return g_fwd_launches; }
int backward_launch_count() { return g_bwd_launches; }


size_t trunk_partial_floats(int Mb, int C) {
  size_t mx = 0;
  for (int mode : {1, 2, 3, 5}) {
    mx = std::max(mx, (size_t)plan_conv1_wgrad(Mb, mode).splits * 257 * 32);
    mx = std::max(mx, (size_t)plan_conv2_wgrad(Mb, mode).splits * 513 * 64);
    mx = std::max(mx, (size_t)plan_conv3_wgrad(Mb, mode).splits * 577 * 64);
  }
  if (C == 1) mx = std::max(mx, (size_t)plan_conv1_wgrad_c1(Mb).splits * 65 * 32);
  return std::max(mx, (size_t)16 * 32 * 256);   // also the scratch of emb_backward (kEmbChunks * A * 256)
}

}  // namespace drl

// The launch plan net_backward / net_forward use at B x T in math mode `mode`, read by the per-kernel tests to assert which
// edges a case reaches (tests/layer_parity.py launch_facts): out[0..2] = split-K count of the conv1 / conv2 / conv3 weight
// gradients, out[3] / out[4] = frames per CTA of the persistent conv1 forward / weight-gradient kernels (math mode 5; 0
// otherwise), out[5] = the M tile of the 16-bit split core (rows per CTA of every GEMM16 launch).
extern "C" int drl_debug_launch_plan(int32_t B, int32_t T, int32_t mode, int32_t* out) {
  using namespace drl;
  if (!out || B < 1 || T < 3) { set_error("launch_plan: need out, B >= 1, T >= 3"); return DRL_ERR_INVALID; }
  const int M = B * T, Mb = B * (T - 2);
  if (mode == 5) {
    const int sms = device_sm_count();
    out[0] = std::min(Mb, sms);                                 // launch_conv1_wgrad_tma: one partial slab per CTA
    out[3] = cdiv(M, std::min(M, sms));
    out[4] = cdiv(Mb, std::min(Mb, sms));
  } else {
    out[0] = plan_conv1_wgrad(Mb, mode).splits;
    out[3] = out[4] = 0;
  }
  out[1] = plan_conv2_wgrad(Mb, mode).splits;
  out[2] = plan_conv3_wgrad(Mb, mode).splits;
  out[5] = X64L2::BM;
  return DRL_OK;
}

namespace drl {
template <class Cfg, class AL, class BL, class EP>
static int umma16_resident_ctas(int32_t* out) {
  using SM = Umma16Smem<Cfg, AL, BL>;
  auto kern = gemm_umma16_kernel<Cfg, AL, BL, EP>;
  int n = 0;
  DRL_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::BYTES));
  DRL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, Cfg::NT, SM::BYTES));
  *out = n;
  return DRL_OK;
}
}  // namespace drl

// The CTAs per SM that the two-CTA-per-SM kernels of math mode 5 actually get (occupancy at the block size and dynamic
// shared memory they launch with): out[0] / out[1] = conv2 / conv3 forward, out[2] = conv2 data gradient.
// A register or shared-memory change that drops one of them to one CTA per SM changes no result, only the step time.
extern "C" int drl_debug_gemm16_residency(int32_t* out) {
  using namespace drl;
  if (!out) { set_error("gemm16_residency: need out"); return DRL_ERR_INVALID; }
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  using FwdB = PretiledB<PlainB>;
  using FwdE = EpBiasAct<true, true>;
  DRL_TRY((umma16_resident_ctas<X64L2, Conv2AP, FwdB, FwdE>(out + 0)));
  DRL_TRY((umma16_resident_ctas<X64L2, Conv3AP, FwdB, FwdE>(out + 1)));
  DRL_TRY((umma16_resident_ctas<X64T2, Conv2DAP, PretiledB<Conv2DBm>, Conv2DEm>(out + 2)));
  return DRL_OK;
}

// Local memory per thread of three math-mode-5 GEMMs of the IMPALA step: out[0] = lstm_fwd, out[1] = lstm_dgrad,
// out[2] = lstm_wgrad.  An accumulator that lands in local memory makes ptxas serialise every wgmma of the main loop:
// the results stay the same, only the kernels get slower.
extern "C" int drl_debug_gemm16_local_bytes(int32_t* out) {
  using namespace drl;
  if (!out) { set_error("gemm16_local_bytes: need out"); return DRL_ERR_INVALID; }
  if (drl_device_count() < 1) { set_error("CUDA device not available (no CPU fallback)"); return DRL_ERR_CUDA; }
  cudaFuncAttributes fa[3];
  DRL_CUDA_CHECK(cudaFuncGetAttributes(&fa[0], gemm_umma16_kernel<X256L, LstmA, PretiledB<PlainB>, EpRaw<false>>));
  DRL_CUDA_CHECK(cudaFuncGetAttributes(&fa[1], gemm_umma16_kernel<X128D, PlainA, PretiledB<PlainBT>, EpLstmDx>));
  DRL_CUDA_CHECK(cudaFuncGetAttributes(&fa[2], gemm_bulk16_kernel<BK256, EpRaw<false>>));
  for (int i = 0; i < 3; ++i) out[i] = (int32_t)fa[i].localSizeBytes;
  return DRL_OK;
}

namespace drl {

size_t lstm_image_bytes(int which, int M, int Mb) {
  (void)M;
  return which == 1 ? operand_image16_bytes<128>(Geo::XK, Mb)     // x^T  (A of lstm_wgrad)
                    : operand_image16_bytes<256>(Geo::G4, Mb);    // dz^T (B of lstm_wgrad)
}

void weight_image_sizes(size_t (&b)[WeightImages::kCount]) {
  b[0] = weight_image_bytes<32>(32, 256);
  b[1] = weight_image_bytes<64>(64, 512);
  b[2] = weight_image_bytes<64>(64, 576);
  b[3] = weight_image_bytes<256>(Geo::G4, Geo::XK);
  b[4] = weight_image_bytes<128>(Geo::FLAT + Geo::EMB, Geo::G4);
  b[5] = weight_image_bytes<256>(576, 64);   // the dCol operands of math modes 2 and 3; larger than the 16-bit dgrad images
  b[6] = weight_image_bytes<256>(512, 64);   // of math mode 5 (weight_image16_bytes<64>(64, 576), <64>(128, 256))
}

// Refresh the weight images (4 launches on the side stream + 1 for the two conv-forward images; ~60 MB written).
// Must run after every parameter change.  Image 0 (conv1) is unused: conv1 is the first kernel of the step and its
// weight tile is 1/5 of a stage.
// math mode 5: the same seven images in the 16-bit K-major form (gemm_umma16.cuh); they fit into the same buffers.
// Images 5 / 6 are the B operands of the conv3 / conv2 data gradients (gather form: B(k = (tap, co), n = ci)).
static int retile_dgrad16(cudaStream_t s, const ParamLayout& pl, const float* P, const WeightImages& wi) {
  DRL_TRY((launch_retile_b16<64, Fmt16>(s, Conv3DB{P + pl.conv3_w}, 64, 576, wi.img[5])));
  DRL_TRY((launch_retile_b16<64, Fmt16>(s, Conv2DBm{{P + pl.conv2_w}}, 128, 256, wi.img[6])));
  return DRL_OK;
}

int net_retile16(cudaStream_t s_rest, const ParamLayout& pl, const float* P, const WeightImages& wi) {
  prof_mark(s_rest, "weight_retile");
  DRL_TRY((launch_retile_b16<256, Fmt16>(s_rest, PlainB{P + pl.lstm_w, Geo::G4, 0}, Geo::G4, Geo::XK, wi.img[3])));
  DRL_TRY((launch_retile_b16<128, Fmt16>(s_rest, PlainBT{P + pl.lstm_w, Geo::G4, 0}, Geo::FLAT + Geo::EMB, Geo::G4, wi.img[4])));
  return retile_dgrad16(s_rest, pl, P, wi);
}

int net_retile(cudaStream_t, cudaStream_t s_rest, const ParamLayout& pl, const float* P, const WeightImages& wi) {
  prof_mark(s_rest, "weight_retile");
  DRL_TRY((launch_retile_b<256>(s_rest, PlainB{P + pl.lstm_w, Geo::G4, 0}, Geo::G4, Geo::XK, wi.img[3])));
  DRL_TRY((launch_retile_b<128>(s_rest, PlainBT{P + pl.lstm_w, Geo::G4, 0}, Geo::FLAT + Geo::EMB, Geo::G4, wi.img[4])));
  return conv_dcol_images_tf32(s_rest, pl, P, wi.img[5], wi.img[6]);
}

int net_forward(const Streams& st, const ParamLayout& pl, const float* P, const WeightImages& wi, const Inputs& in,
                const Acts& act, int B, int T, int mode, bool retile, const Recurrence& rec) {
  const int M = B * T;
  const RowMap map{B, T};
  int n = 0, nsplit = 4;
  cudaStream_t s = st.main;
  const cudaStream_t side = st.par ? st.side : st.main;
  // action embedding table (:12-16): only A distinct inputs exist; depends on parameters only -> side stream
  DRL_TRY(fork_to_side(st, 0));
  s = side;
  // weight images of this step's parameters, all on the side stream: the conv2/conv3 forward ones first (main waits
  // for them behind conv1), the LSTM / dgrad ones behind the embedding table (joined before lstm_fwd)
  const bool m16 = mode == 5;
  bool c3_event = false;   // conv3's weight image has its own event (math mode 5)
  // math mode 5: conv1 is the frame-resident TMA kernel (conv1_tma.cuh), which builds its 32 KB weight image itself
  if (retile && m16) {
    prof_mark(s, "weight_retile");
    DRL_TRY((launch_retile_b16<64, Fmt16>(s, PlainB{P + pl.conv2_w, 64, 0}, 64, 512, wi.img[1])));
    if (st.par) DRL_CUDA_CHECK(cudaEventRecord(st.ev[7], side));          // conv2 image (main waits behind conv1)
    DRL_TRY((launch_retile_b16<64, Fmt16>(s, PlainB{P + pl.conv3_w, 64, 0}, 64, 576, wi.img[2])));
    if (st.par) DRL_CUDA_CHECK(cudaEventRecord(st.ev[4], side));          // conv3 image (main waits behind conv2)
    c3_event = st.par;
    n += 2;
  } else if (retile && mode >= 2) {
    prof_mark(s, "weight_retile");
    DRL_TRY(conv_images_tf32(s, pl, P, wi.img[1], wi.img[2]));
    n += 2;
    if (st.par) DRL_CUDA_CHECK(cudaEventRecord(st.ev[7], side));
  }
  KERNEL("emb_fwd",
         emb_forward(s, P + pl.emb1_w, P + pl.emb1_b, P + pl.emb2_w, P + pl.emb2_b, act.e1, act.table, pl.A), 1);
  s = st.main;
  bool late_images = false;   // side still carries the images only the backward pass reads when lstm_fwd is enqueued
  if (retile && mode >= 2) {
    if (m16 && st.par) {
      // the LSTM forward image first; lstm_fwd waits for it (and the embedding table) only -- the three images of the
      // backward pass (LSTM dgrad, conv3 / conv2 dgrad) are joined at the end of the forward pass, long after they are done
      prof_mark(side, "weight_retile");
      DRL_TRY((launch_retile_b16<256, Fmt16>(side, PlainB{P + pl.lstm_w, Geo::G4, 0}, Geo::G4, Geo::XK, wi.img[3])));
      DRL_CUDA_CHECK(cudaEventRecord(st.ev[1], side));
      late_images = true;   // LSTM dgrad + two conv dgrad images: behind lstm_gates_fwd, in the shadow of the small head kernels
    } else if (m16) {
      DRL_TRY(net_retile16(side, pl, P, wi));
    } else {
      DRL_TRY(net_retile(st.main, side, pl, P, wi));
    }
    n += 4;
  }
  // attention_CNN (model/impala_actor_critic.py:6-10): u8 frames -> a1 [M,20,20,32] -> a2 [M,9,9,64] -> a3 [M,7,7,64]
  // = flatten HWC [M,3136]; conv2 waits for its weight image, conv3 for its own in math mode 5
  if (m16) {
    // a1 and a2 are written with their 16-bit planes, from which conv2 / conv3 copy their A tiles
    const size_t n1 = (size_t)M * 400 * 32, n2 = (size_t)M * 81 * 64;
    prof_mark(s, "conv1_fwd");
    DRL_TRY(launch_conv1_fwd_tma(s, in.frames, M, map, P + pl.conv1_w,
                                 EpConv1{act.a1, 32, P + pl.conv1_b, Plane16{act.a1p, n1}}));
    ++n;
    if (retile && st.par) DRL_CUDA_CHECK(cudaStreamWaitEvent(st.main, st.ev[7], 0));
    {
      Conv2AP al{Conv2A{act.a1, map}, act.a1, act.a1p, n1};
      PretiledB<PlainB> blp{wi.img[1], 512 / 64};
      EpBiasAct<true, true> ep{act.a2, 64, 0, P + pl.conv2_b, 0, 1.0f, Plane16{act.a2p, n2}};
      GEMM16("conv2_fwd", X64L2, al, blp, ep, M * 81, 64, 512, 1, 512, 0);
    }
    if (c3_event) DRL_CUDA_CHECK(cudaStreamWaitEvent(st.main, st.ev[4], 0));
    {
      Conv3AP al{Conv3A{act.a2, map}, act.a2, act.a2p, n2};
      PretiledB<PlainB> blp{wi.img[2], 576 / 64};
      EpBiasAct<true, true> ep{act.a3, 64, 0, P + pl.conv3_b, 0, 1.0f};
      GEMM16("conv3_fwd", X64L2, al, blp, ep, M * 49, 64, 576, 1, 576, 0);
    }
  } else {
    const cudaEvent_t images_ready = retile && mode >= 2 && st.par ? st.ev[7] : nullptr;
    DRL_TRY(conv_forward_tf32<Geo::IC>(s, pl, P, wi.img[1], wi.img[2], in.frames, B, T, act.a1, act.a2, act.a3, mode,
                                        false, images_ready, &n));
  }
  if (late_images) DRL_CUDA_CHECK(cudaStreamWaitEvent(st.main, st.ev[1], 0));
  else DRL_TRY(join_from_side(st, 1));
  // LSTM pre-activation z = [a3 | emb | h0] W  (split-K partial sums; bias added in the gate kernel) (:18-25).
  // Recurrent mode: only the K = 3392 input rows, [a3 | emb] W[:3392]; the h rows multiply inside the recurrence.
  {
    LstmA al{act.a3, act.table, in.pa, in.h0, map};
    PlainB bl{P + pl.lstm_w, Geo::G4, 0};
    EpRaw<false> ep{act.zpart, Geo::G4, (size_t)M * Geo::G4, 1.0f, 0, Geo::G4};
    // FFMA: 4 splits of 57 x 16.  Tensor cores: 128 x 256 tiles -> 5 x 4 output tiles x 7 splits of 17 x 32 (B = 32, T = 20)
    // Recurrent mode (math modes 2 and 5): 7 splits of 512 = 8 K tiles of 64 or 16 of 32 (the last 320)
    nsplit = (mode >= 2) ? 7 : 4;
    const int K = rec.on() ? Geo::FLAT + Geo::EMB : Geo::XK;
    const int kchunk = rec.on() ? 512 : m16 ? 576 : (mode >= 2) ? 544 : Geo::XK / 4;   // 16-bit: 9 K tiles of 64 per split
    PretiledB<PlainB> blp{wi.img[3], m16 ? Geo::XK / 64 : Geo::XK / 32};
    if (m16) GEMM16("lstm_fwd", X256L, al, blp, ep, M, Geo::G4, K, nsplit, kchunk, kchunk);
    else GEMM_W("lstm_fwd", CfgMid, U256L, al, bl, blp, ep, M, Geo::G4, K, nsplit, kchunk, kchunk);
  }
  if (rec.on()) {
    KERNEL("lstm_x_reduce", splitk_reduce(s, act.zpart, (size_t)M * Geo::G4, nsplit, act.zx, (size_t)M * Geo::G4), 1);
    prof_mark(s, "lstm_unroll_fwd");
    DRL_CUDA_CHECK(launch_cluster_k(impala_lstm_fwd_cluster_kernel, ImpClu::CL, recurrence_grid(B, rec.clusters_fwd),
                                    ImpClu::T, ImpClu::kFwdSmem, s, act.zx, P + pl.lstm_b,
                                    P + pl.lstm_w + (size_t)(Geo::FLAT + Geo::EMB) * Geo::G4, in.h0, in.c0, in.done,
                                    act.gates, act.tc1, act.h1, act.hin, act.cin, act.c1, B, T));
    ++n;
  } else {
    KERNEL("lstm_gates_fwd",
           lstm_gates_forward(s, act.zpart, nsplit, P + pl.lstm_b, in.c0, act.gates, act.c1, act.tc1, act.h1, M, B,
                              T), 1);
  }
  // heads (fully_connected, :27-30,40-41): z = 0 actor, z = 1 critic
  const size_t head_stride = (size_t)(pl.critic1_w - pl.actor1_w);
  if (late_images) {
    // the three images only the backward pass reads (~25 us of memory-bound work) would compete with conv2_fwd / conv3_fwd
    // for the SMs if launched with the others; the head layers that follow leave most of the GPU idle
    DRL_TRY(fork_to_side(st, 3));
    DRL_TRY((launch_retile_b16<128, Fmt16>(side, PlainBT{P + pl.lstm_w, Geo::G4, 0}, Geo::FLAT + Geo::EMB, Geo::G4, wi.img[4])));
    DRL_TRY(retile_dgrad16(side, pl, P, wi));
  }
  {
    PlainA al{act.h1, Geo::L, 0};
    PlainB bl{P + pl.actor1_w, Geo::HID, head_stride};
    EpBiasAct<true, true> ep{act.hid1, Geo::HID, (size_t)M * Geo::HID, P + pl.actor1_b, head_stride, 1.0f};
    if (m16) GEMM16("heads_l1_fwd", XH, al, bl, ep, M, Geo::HID, Geo::L, 2, Geo::L, 0);
    else GEMM_FFMA("heads_l1_fwd", CfgSmall, al, bl, ep, M, Geo::HID, Geo::L, 2, Geo::L, 0);
  }
  {
    PlainA al{act.hid1, Geo::HID, (size_t)M * Geo::HID};
    PlainB bl{P + pl.actor2_w, Geo::HID, head_stride};
    EpBiasAct<true, true> ep{act.hid2, Geo::HID, (size_t)M * Geo::HID, P + pl.actor2_b, head_stride, 1.0f};
    if (m16) GEMM16("heads_l2_fwd", XH, al, bl, ep, M, Geo::HID, Geo::HID, 2, Geo::HID, 0);
    else GEMM_FFMA("heads_l2_fwd", CfgSmall, al, bl, ep, M, Geo::HID, Geo::HID, 2, Geo::HID, 0);
  }
  KERNEL("heads_out_fwd",
         heads_out_forward(s, act.hid2, act.hid2 + (size_t)M * Geo::HID, P + pl.actor3_w, P + pl.actor3_b,
                           P + pl.critic3_w, P + pl.critic3_b, act.logits, act.policy, act.value, M, pl.A), 1);
  if (late_images) DRL_TRY(join_from_side(st, 1));   // the backward images: done ~70 us ago, keeps net_forward self-contained
  g_fwd_launches = n;
  return DRL_OK;
}

// The convolutions of the policy engine (policy.cu): the math-mode-5 kernels and launch configurations of net_forward
// over n single frames (B = n, T = 1), on one stream.  The conv2 / conv3 weight images are the engine's own and are
// rebuilt by conv_images16 whenever its parameters change.
int conv_images16(cudaStream_t s, const ParamLayout& pl, const float* P, uint8_t* img_conv2, uint8_t* img_conv3) {
  DRL_TRY((launch_retile_b16<64, Fmt16>(s, PlainB{P + pl.conv2_w, 64, 0}, 64, 512, img_conv2)));
  DRL_TRY((launch_retile_b16<64, Fmt16>(s, PlainB{P + pl.conv3_w, 64, 0}, 64, 576, img_conv3)));
  return DRL_OK;
}

int conv_forward16(cudaStream_t s, const ParamLayout& pl, const float* P, const uint8_t* img_conv2,
                   const uint8_t* img_conv3, const uint8_t* frames, int n, float* a1, float* a2, float* a3,
                   uint16_t* a1p, uint16_t* a2p) {
  const RowMap map{n, 1};
  const size_t n1 = (size_t)n * 400 * 32, n2 = (size_t)n * 81 * 64;
  DRL_TRY(launch_conv1_fwd_tma(s, frames, n, map, P + pl.conv1_w, EpConv1{a1, 32, P + pl.conv1_b, Plane16{a1p, n1}}));
  {
    Conv2AP al{Conv2A{a1, map}, a1, a1p, n1};
    PretiledB<PlainB> blp{img_conv2, 512 / 64};
    EpBiasAct<true, true> ep{a2, 64, 0, P + pl.conv2_b, 0, 1.0f, Plane16{a2p, n2}};
    DRL_TRY((launch_gemm_umma16<X64L2>(s, al, blp, ep, n * 81, 64, 512, 1, 512, 0)));
  }
  {
    Conv3AP al{Conv3A{a2, map}, a2, a2p, n2};
    PretiledB<PlainB> blp{img_conv3, 576 / 64};
    EpBiasAct<true, true> ep{a3, 64, 0, P + pl.conv3_b, 0, 1.0f};
    DRL_TRY((launch_gemm_umma16<X64L2>(s, al, blp, ep, n * 49, 64, 576, 1, 576, 0)));
  }
  return DRL_OK;
}

// The conv trunk backward of math mode 5, the same steps, streams and events as conv_backward_tf32 (layer_defs.cuh) on
// the 16-bit split core: weight gradients from two gathered operands, data gradients in gather form, the frame-resident
// TMA kernel for conv1's weight gradient.
static int conv_backward16(const Streams& st, const ParamLayout& pl, const WeightImages& wi, float* G,
                           const uint8_t* frames, int B, int T, const Acts& act, const Bwd& bw, int* launches) {
  const int mode = 5, M = B * T, Mb = B * (T - 2);
  const RowMap map{B, T};
  cudaStream_t s = st.par ? st.side : st.main;
  int n = 0;
  {
    const SplitPlan sp = plan_conv3_wgrad(Mb, mode);
    const size_t slab = 577 * 64;
    Conv3WA al{act.a2, map};
    PlainB bl{bw.da3, 64, 0};
    EpRaw<true> ep{bw.wg_part, 64, slab, 1.0f, 576, 64};
    GEMM16("conv3_wgrad", X64W8x2, al, bl, ep, 576, 64, Mb * 49, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv3_wgrad_reduce", splitk_reduce(s, bw.wg_part, slab, sp.splits, G + pl.conv3_w, slab), 1);
  }
  s = st.main;
  {
    // gather form: rows = input pixels, K = 9 taps x 64 output channels (taps outside the output are zero), ReLU mask of
    // a2 in the epilogue; each tap's partial sum is rounded to fp32 and the taps are added in (ky, kx) order, as
    // col2im_conv3 adds the dCol of math modes 2 and 3: the same da2, bit for bit
    Conv3DAP al{Conv3DA{bw.da3}, bw.da3, bw.da3p, (size_t)Mb * Geo::FLAT};
    PretiledB<Conv3DB> blp{wi.img[5], 576 / 64};
    Conv3DE ep{bw.da2, act.a2, Plane16{bw.da2p, (size_t)Mb * 81 * 64}};
    GEMM16("conv3_dgrad", X64T2, al, blp, ep, Mb * 81, 64, 576, 1, 576, 0);
  }
  DRL_TRY(fork_to_side(st, 5));
  s = st.par ? st.side : st.main;
  {
    const SplitPlan sp = plan_conv2_wgrad(Mb, mode);
    const size_t slab = 513 * 64;
    Conv2WA al{act.a1, map};
    PlainB bl{bw.da2, 64, 0};
    EpRaw<true> ep{bw.wg_part, 64, slab, 1.0f, 512, 64};
    GEMM16("conv2_wgrad", X64W8x2, al, bl, ep, 512, 64, Mb * 81, sp.splits, sp.kchunk, sp.kchunk);
    KERNEL("conv2_wgrad_reduce", splitk_reduce(s, bw.wg_part, slab, sp.splits, G + pl.conv2_w, slab), 1);
  }
  s = st.main;
  {
    // merged-phase gather form: row = the 2 x 2 block of input pixels (2i + py, 2j + px); all four parity classes read
    // the same dY taps (i - a, j - b), so K = (a, b, co) = 256 and N = (py, px, ci) = 128, in two N tiles (py = 0, 1);
    // ReLU mask of a1 in the epilogue; per-tap partial sums added in (a, b) order, as in col2im_conv2
    Conv2DAP al{Conv2DA{bw.da2}, bw.da2, bw.da2p, (size_t)Mb * 81 * 64};
    PretiledB<Conv2DBm> blp{wi.img[6], 256 / 64};
    Conv2DEm ep{{bw.da1, act.a1}};
    GEMM16("conv2_dgrad", X64T2, al, blp, ep, Mb * 100, 128, 256, 1, 256, 0);
  }
  // conv1 (input is data: weight gradient only): one partial slab per CTA, then the fixed-order reduce
  const size_t slab = 257 * 32;
  int splits = 0;
  prof_mark(s, "conv1_wgrad");
  DRL_TRY(launch_conv1_wgrad_tma(s, frames, M, Mb, map, bw.da1, bw.wg_part2, bw.wg_part_floats, &splits));
  ++n;
  KERNEL("conv1_wgrad_reduce", splitk_reduce(s, bw.wg_part2, slab, splits, G + pl.conv1_w, slab), 1);
  *launches += n;
  return DRL_OK;
}

int net_backward(const Streams& st, const ParamLayout& pl, const float* P, const WeightImages& wi, float* G,
                 const Inputs& in, const Acts& act, const Bwd& bw, int B, int T, int mode, const Recurrence& rec) {
  const bool m16 = mode == 5;
  cudaStream_t s = st.main;
  const cudaStream_t side = st.par ? st.side : st.main;
  const int M = B * T;
  const int Mb = B * (T - 2);   // rows t <= T-3 are the contiguous prefix (time-major)
  const RowMap map{B, T};
  const size_t head_stride = (size_t)(pl.critic1_w - pl.actor1_w);
  const int A = pl.A;
  int n = 0;

  // ---- heads -------------------------------------------------------------------------------
  KERNEL("heads_out_bwd",
         heads_out_backward(s, bw.dlogits, bw.dv, P + pl.actor3_w, P + pl.critic3_w, act.hid2,
                            act.hid2 + (size_t)M * Geo::HID, bw.dhid2, bw.dhid2 + (size_t)Mb * Geo::HID, Mb, A), 1);
  if (m16) {
    // x^T as an operand image (A of lstm_wgrad): depends on the forward pass only -> side stream, in the shadow of the
    // small head kernels
    DRL_TRY(fork_to_side(st, 0));
    prof_mark(side, "lstm_xt_image");
    if (rec.on())
      DRL_TRY((launch_retile_t16<128, Fmt16>(side, LstmHinAT{act.a3, act.table, in.pa, act.hin, map, Geo::L}, Geo::XK, Mb,
                                             act.img_xt)));
    else
      DRL_TRY((launch_retile_t16<128, Fmt16>(side, LstmAT{act.a3, act.table, in.pa, in.h0, map}, Geo::XK, Mb, act.img_xt)));
    ++n;
  }
  // dlogits / dv / dhid2 are ready: three weight gradients can start beside the chain (on the second side lane if any)
  const bool lane2 = st.par && st.side2 != nullptr;
  const cudaStream_t small = lane2 ? st.side2 : side;
  if (lane2) DRL_TRY(fork_to_side2(st, 0));
  else DRL_TRY(fork_to_side(st, 0));
  s = small;
  {  // d actor3 [256(+1), A]
    PlainAT al{act.hid2, Geo::HID, 0};
    PlainB bl{bw.dlogits, 32, 0};
    EpRaw<true> ep{G + pl.actor3_w, A, 0, 1.0f, Geo::HID, A};
    GEMM_FFMA_KS("actor3_wgrad", CfgSmall, 3, al, bl, ep, Geo::HID, 32, Mb, 1, Mb, 0);
  }
  {  // d critic3 [256(+1), 1]
    PlainAT al{act.hid2 + (size_t)M * Geo::HID, Geo::HID, 0};
    PlainB bl{bw.dv, 32, 0};
    EpRaw<true> ep{G + pl.critic3_w, 1, 0, 1.0f, Geo::HID, 1};
    GEMM_FFMA_KS("critic3_wgrad", CfgSmall, 3, al, bl, ep, Geo::HID, 32, Mb, 1, Mb, 0);
  }
  {  // d {actor2, critic2} = hid1^T dhid2
    PlainAT al{act.hid1, Geo::HID, (size_t)M * Geo::HID};
    PlainB bl{bw.dhid2, Geo::HID, (size_t)Mb * Geo::HID};
    EpRaw<true> ep{G + pl.actor2_w, Geo::HID, head_stride, 1.0f, Geo::HID, Geo::HID};
    GEMM_FFMA_KS("heads_l2_wgrad", CfgSmall, 3, al, bl, ep, Geo::HID, Geo::HID, Mb, 2, Mb, 0);
  }
  s = st.main;
  {  // dhid1 = dhid2 W2^T * relu'(hid1)
    PlainA al{bw.dhid2, Geo::HID, (size_t)Mb * Geo::HID};
    PlainBT bl{P + pl.actor2_w, Geo::HID, head_stride};
    EpReluMask ep{bw.dhid1, act.hid1, Geo::HID, (size_t)Mb * Geo::HID, (size_t)M * Geo::HID};
    if (m16) GEMM16("heads_l2_dgrad", XH, al, bl, ep, Mb, Geo::HID, Geo::HID, 2, Geo::HID, 0);
    else GEMM_FFMA_KS("heads_l2_dgrad", CfgSmall, 4, al, bl, ep, Mb, Geo::HID, Geo::HID, 2, Geo::HID, 0);
  }
  if (lane2) DRL_TRY(fork_to_side2(st, 1));
  else DRL_TRY(fork_to_side(st, 2));
  s = small;
  {  // d {actor1, critic1} = h1^T dhid1
    PlainAT al{act.h1, Geo::L, 0};
    PlainB bl{bw.dhid1, Geo::HID, (size_t)Mb * Geo::HID};
    EpRaw<true> ep{G + pl.actor1_w, Geo::HID, head_stride, 1.0f, Geo::L, Geo::HID};
    GEMM_FFMA_KS("heads_l1_wgrad", CfgSmall, 3, al, bl, ep, Geo::L, Geo::HID, Mb, 2, Mb, 0);
  }
  s = st.main;
  {  // dh1 contributions (actor, critic) = dhid1 W1^T ; summed in the gate kernel
    PlainA al{bw.dhid1, Geo::HID, (size_t)Mb * Geo::HID};
    PlainBT bl{P + pl.actor1_w, Geo::HID, head_stride};
    EpRaw<false> ep{bw.dh_part, Geo::L, (size_t)Mb * Geo::L, 1.0f, 0, Geo::L};
    if (m16) GEMM16("heads_l1_dgrad", XH, al, bl, ep, Mb, Geo::L, Geo::HID, 2, Geo::HID, 0);
    else GEMM_FFMA_KS("heads_l1_dgrad", CfgSmall, 4, al, bl, ep, Mb, Geo::L, Geo::HID, 2, Geo::HID, 0);
  }
  // ---- LSTM cell ---------------------------------------------------------------------------
  if (rec.on()) {
    prof_mark(s, "lstm_unroll_bwd");
    DRL_CUDA_CHECK(launch_cluster_k(impala_lstm_bwd_cluster_kernel, ImpClu::CL, recurrence_grid(B, rec.clusters_bwd),
                                    ImpClu::T, ImpClu::kBwdSmem, s, bw.dh_part, (size_t)Mb * Geo::L, act.gates, act.tc1,
                                    act.cin, P + pl.lstm_w + (size_t)(Geo::FLAT + Geo::EMB) * Geo::G4, in.done, bw.dz, B,
                                    T));
    ++n;
  } else {
    KERNEL("lstm_gates_bwd",
           lstm_gates_backward(s, bw.dh_part, (size_t)Mb * Geo::L, act.gates, act.tc1, in.c0, bw.dz, Mb, B, T), 1);
  }
  DRL_TRY(fork_to_side(st, 3));
  s = side;
  {  // d lstm kernel [3648(+1), 1024] = x^T dz ; bias gradient = column sums of dz
    PlainB bl{bw.dz, Geo::G4, 0};
    if (m16) {
      const int ktm = cdiv(Mb, 64);
      prof_mark(s, "lstm_dzt_image");
      DRL_TRY((launch_retile_t16<256, Fmt16>(s, bl, Geo::G4, Mb, bw.img_dzt)));
      // bias gradient = column sums of dz (row XK of [w; b]), fixed order
      DRL_TRY(splitk_reduce(s, bw.dz, Geo::G4, Mb, G + pl.lstm_w + (size_t)Geo::XK * Geo::G4, Geo::G4));
      prof_mark(s, "lstm_wgrad");
      EpRaw<false> epw{G + pl.lstm_w, Geo::G4, 0, 1.0f, Geo::XK, Geo::G4};
      DRL_TRY((launch_gemm_bulk16<BK256>(s, ImageOp{act.img_xt, ktm}, ImageOp{bw.img_dzt, ktm}, epw, Geo::XK, Geo::G4, Mb,
                                         1, Mb, 0)));
      n += 3;
    } else if (rec.on()) {
      LstmHinAT al{act.a3, act.table, in.pa, act.hin, map, Geo::L};
      EpRaw<true> ep{G + pl.lstm_w, Geo::G4, 0, 1.0f, Geo::XK, Geo::G4};
      GEMM("lstm_wgrad", CfgBig, U256, al, bl, ep, Geo::XK, Geo::G4, Mb, 1, Mb, 0);
    } else {
      LstmAT al{act.a3, act.table, in.pa, in.h0, map};
      EpRaw<true> ep{G + pl.lstm_w, Geo::G4, 0, 1.0f, Geo::XK, Geo::G4};
      GEMM("lstm_wgrad", CfgBig, U256, al, bl, ep, Geo::XK, Geo::G4, Mb, 1, Mb, 0);   // 29 x 4 = 116 CTAs: one wave
    }
    // the head gradients (earlier on this stream, or on the second lane: joined here) and the LSTM gradient are now
    // in the bucket: [lstm_w .. end)
    if (lane2) DRL_TRY(join_side2_into(st, 2, side));
    if (st.par && st.ev_lstm_grads) DRL_CUDA_CHECK(cudaEventRecord(st.ev_lstm_grads, side));
  }
  s = st.main;
  {  // d[a3 | emb] = dz W[:3392]^T  (h0, c0 are fed data: no gradient, agent/impala.py:38-39)
    PlainA al{bw.dz, Geo::G4, 0};
    PlainBT bl{P + pl.lstm_w, Geo::G4, 0};
    EpLstmDx ep{bw.da3, act.a3, bw.du, Plane16{bw.da3p, (size_t)Mb * Geo::FLAT}};   // plane: math mode 5 only
    PretiledB<PlainBT> blp{wi.img[4], m16 ? Geo::G4 / 64 : Geo::G4 / 32};
    if (m16) GEMM16("lstm_dgrad", X128D, al, blp, ep, Mb, Geo::FLAT + Geo::EMB, Geo::G4, 1, Geo::G4, 0);
    else GEMM_W("lstm_dgrad", CfgMid, U128L, al, bl, blp, ep, Mb, Geo::FLAT + Geo::EMB, Geo::G4, 1, Geo::G4, 0);
  }
  // ---- action embedding + conv3 weight gradient (side) -------------------------------------
  // the embedding gradient: four small kernels that the hardware schedules late behind the big GEMMs (32 us alone, ~80 us
  // in the graph).  On one GPU they stay in front of conv3_wgrad on `side` (the second lane measured 0.4 % slower: the
  // backward pass is throughput-bound, earlier weight gradients only take SMs from the main chain).  With the fused peer
  // exchange the side stream IS the tail of the step (the early exchange part competes with it), and moving them to the
  // second lane (own scratch) gains 1 % at 2 GPUs.
  const bool emb2 = lane2 && bw.emb_scratch != nullptr && st.ev_lstm_grads != nullptr;
  if (emb2) {
    DRL_TRY(fork_to_side2(st, 3));
    s = st.side2;
    KERNEL("emb_bwd",
           emb_backward(s, bw.du, in.pa, act.e1, act.table, P + pl.emb2_w, bw.dpre2, bw.dpre1, G + pl.emb1_w,
                        G + pl.emb1_b, G + pl.emb2_w, G + pl.emb2_b, bw.emb_scratch, Mb, B, T, A), 4);
  }
  DRL_TRY(fork_to_side(st, 4));
  s = side;
  if (!emb2)
    KERNEL("emb_bwd",
           emb_backward(s, bw.du, in.pa, act.e1, act.table, P + pl.emb2_w, bw.dpre2, bw.dpre1, G + pl.emb1_w,
                        G + pl.emb1_b, G + pl.emb2_w, G + pl.emb2_b, bw.wg_part, Mb, B, T, A), 4);
  // ---- conv trunk --------------------------------------------------------------------------
  if (m16) DRL_TRY(conv_backward16(st, pl, wi, G, in.frames, B, T, act, bw, &n));
  else DRL_TRY(conv_backward_tf32<Geo::IC>(st, pl, P, wi, G, in.frames, map, Mb, act, bw, mode, &n));
  if (lane2) DRL_TRY(join_side2_into(st, 2, st.main));
  DRL_TRY(join_from_side(st, 6));
  g_bwd_launches = n;
  return DRL_OK;
}

}  // namespace drl
