// The U-Net handle (shared by the forward plan, unet.cu, and the backward plan, unet_bwd.cu).
#pragma once
#include "net.cuh"

struct b200ad_unet : b200ad::NetBase {
  b200ad_unet_config cfg;
  std::vector<b200ad::Block> blocks;
};
