// The U-Net handle (shared by the forward plan, unet.cu, and the backward plan, backward.cu).
#pragma once
#include "net.cuh"

struct b200ad_unet : b200ad::NetBase {   // one model part: parts[0]
  b200ad_unet_config cfg;
};

namespace b200ad {
Plan build_plan(const b200ad_unet* h, uint8_t* ws_base, int N, int H, int W);   // the forward plan (null: sizes only)
}
