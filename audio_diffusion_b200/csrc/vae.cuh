// The autoencoder handle (shared by the forward plans, vae.cu, and the backward plans, unet_bwd.cu).
#pragma once
#include "net.cuh"

struct b200ad_vae : b200ad::NetBase {
  b200ad_vae_config cfg;
  std::vector<b200ad::Block> enc, dec;   // encoder, decoder
};

namespace b200ad {
enum { ENC = 0, DEC = 1 };               // the two plans (forward and backward)
}
