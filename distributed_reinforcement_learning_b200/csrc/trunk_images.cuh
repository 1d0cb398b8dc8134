// trunk_images.cuh -- the weight images of the attention_CNN in math modes 2 and 3, built by every learner (layers.cu,
// apex.cu, r2d2.cu) and by the Ape-X / R2D2 target refresh (adam_learner.cu).  Templates over the layout (any layout
// with conv2_w / conv3_w offsets), so that only the translation units that call them instantiate retile_b_kernel.
#pragma once
#include "gemm_umma.cuh"
#include "loaders.cuh"

namespace drl {

// the conv2 / conv3 forward images (WeightImages slots 1 and 2)
template <class Layout>
int conv_images_tf32(cudaStream_t s, const Layout& pl, const float* P, uint8_t* img_conv2, uint8_t* img_conv3) {
  DRL_TRY((launch_retile_b<64>(s, PlainB{P + pl.conv2_w, 64, 0}, 64, 512, img_conv2)));
  DRL_TRY((launch_retile_b<64>(s, PlainB{P + pl.conv3_w, 64, 0}, 64, 576, img_conv3)));
  return DRL_OK;
}

// the B operands of the conv3 / conv2 dCol GEMMs of the data gradients (WeightImages slots 5 and 6)
template <class Layout>
int conv_dcol_images_tf32(cudaStream_t s, const Layout& pl, const float* P, uint8_t* img_conv3, uint8_t* img_conv2) {
  DRL_TRY((launch_retile_b<256>(s, PlainBT{P + pl.conv3_w, 64, 0}, 576, 64, img_conv3)));
  DRL_TRY((launch_retile_b<256>(s, PlainBT{P + pl.conv2_w, 64, 0}, 512, 64, img_conv2)));
  return DRL_OK;
}

}  // namespace drl
