// The autoencoder handle (shared by the forward plans, vae.cu, and the backward plans, backward.cu).
#pragma once
#include "net.cuh"

struct b200ad_vae : b200ad::NetBase {    // two model parts: parts[ENC], parts[DEC]
  b200ad_vae_config cfg;
};

namespace b200ad {
enum { ENC = 0, DEC = 1 };               // the two parts: block lists and plans (forward and backward)
Plan vae_build_plan(const b200ad_vae* h, uint8_t* ws_base, int N, int H, int W);   // both forward plans (null: sizes only)
}
