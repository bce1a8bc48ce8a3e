// Tap sets of the implicit-GEMM convolution: for every way a conv K-segment reads its source, the weight taps to pack, the
// window offset (dh, dw) of each tap relative to the output pixel, and the weight-gradient slot each tap accumulates into.
// The model plans (net.cuh, unet_bwd.cu) and the op-level entry points (api.cu) build their segments from these. Host only.
#pragma once
#include "conv_tc.cuh"
#include "kernels.cuh"

namespace b200ad {

struct TapSet {
  PackTaps pack;
  signed char dh[CONV_MAXTAPS], dw[CONV_MAXTAPS];
  int wtap[CONV_MAXTAPS];  // tap index (kh * K + kw) of the weight gradient; folded taps: the folded tap's own index
};

// ---- forward
// stride-1 KxK conv (K = 1 or 3), padding K / 2
inline TapSet taps_conv(int K) {
  TapSet t{};
  t.pack.ntaps = K * K;
  for (int k = 0; k < K * K; ++k) {
    t.pack.kh[k] = k / K; t.pack.kw[k] = k % K;
    t.dh[k] = (signed char)(k / K - K / 2); t.dw[k] = (signed char)(k % K - K / 2);
    t.wtap[k] = k;
  }
  return t;
}
// Downsample2D(padding 1): stride-2 3x3 conv on parity plane (a, b) of the input, the taps that read rows of parity a and
// columns of parity b; plane pixel (y, x) = input (2y + a, 2x + b), so tap kh reads plane row y - 1 if kh == 0, else y.
inline TapSet taps_parity(int a, int b) {
  TapSet t{};
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw)
      if ((kh != 1) == a && (kw != 1) == b) {
        const int n = t.pack.ntaps++;
        t.pack.kh[n] = kh; t.pack.kw[n] = kw;
        t.dh[n] = kh == 0 ? -1 : 0; t.dw[n] = kw == 0 ? -1 : 0;
        t.wtap[n] = kh * 3 + kw;
      }
  return t;
}
// Downsample2D(padding 0) of the autoencoder: F.pad(x, (0,1,0,1)) then a stride-2 3x3 conv without padding, i.e.
// out[y][x] = sum w[kh][kw] * in[2y+kh][2x+kw].  On parity plane (a, b) that is the taps with kh % 2 == a, kw % 2 == b read
// at row offset kh / 2, column offset kw / 2.
inline TapSet taps_parity_asym(int a, int b) {
  TapSet t{};
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw)
      if ((kh & 1) == a && (kw & 1) == b) {
        const int n = t.pack.ntaps++;
        t.pack.kh[n] = kh; t.pack.kw[n] = kw;
        t.dh[n] = (signed char)(kh >> 1); t.dw[n] = (signed char)(kw >> 1);
        t.wtap[n] = kh * 3 + kw;
      }
  return t;
}
// nearest-2x upsample + 3x3 conv, output parity (a, b): a 2x2 conv on the low-res input whose taps are sums of the 3x3
// taps that read the same low-res pixel. Row taps: a = 0 -> dh = -1 (kh 0), dh = 0 (kh 1,2); a = 1 -> dh = 0 (kh 0,1), +1 (kh 2).
inline TapSet taps_up2(int a, int b) {
  TapSet u{};
  u.pack.fold = 1;
  u.pack.ntaps = 4;
  for (int ri = 0; ri < 2; ++ri)
    for (int ci = 0; ci < 2; ++ci) {
      const int t = ri * 2 + ci;
      const int dh = (a == 0) ? ri - 1 : ri, dw = (b == 0) ? ci - 1 : ci;
      u.dh[t] = (signed char)dh; u.dw[t] = (signed char)dw;
      u.wtap[t] = t;
      unsigned mask = 0;
      for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) {
          const int rdh = (a == 0) ? (kh == 0 ? -1 : 0) : (kh == 2 ? 1 : 0);
          const int rdw = (b == 0) ? (kw == 0 ? -1 : 0) : (kw == 2 ? 1 : 0);
          if (rdh == dh && rdw == dw) mask |= 1u << (kh * 3 + kw);
        }
      u.pack.fold_mask[t] = mask;
    }
  return u;
}

// ---- backward (data gradients: transposed packs, the GEMM output channels are the layer's input channels)
// stride-1 KxK conv: the taps mirrored
inline TapSet taps_mirrored(int K) {
  TapSet t = taps_conv(K);
  t.pack.transpose = 1;
  for (int k = 0; k < K * K; ++k) { t.pack.kh[k] = K - 1 - k / K; t.pack.kw[k] = K - 1 - k % K; }
  return t;
}
// Downsample2D(padding 1): input parity (a, b) <- the taps of matching parity, from the low-res gradient
// (a = 0: kh 1 at dh 0;  a = 1: kh 0 at dh +1, kh 2 at dh 0)
inline TapSet taps_scatter2(int a, int b) {
  TapSet t{};
  t.pack.transpose = 1;
  const int khs[2][2] = {{1, -1}, {0, 2}};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) {
      const int kh = khs[a][i], kw = khs[b][j];
      if (kh < 0 || kw < 0) continue;
      const int n = t.pack.ntaps++;
      t.pack.kh[n] = kh; t.pack.kw[n] = kw;
      t.dh[n] = kh == 0 ? 1 : 0; t.dw[n] = kw == 0 ? 1 : 0;
    }
  return t;
}
// Downsample2D(padding (0, 1, 0, 1)) of the autoencoder: input parity (a, b) <- the taps of matching parity
// (a = 0: kh 0 at dh 0, kh 2 at dh -1;  a = 1: kh 1 at dh 0).  The padded row and column receive no gradient.
inline TapSet taps_scatter2_asym(int a, int b) {
  TapSet t{};
  t.pack.transpose = 1;
  const int khs[2][2] = {{0, 2}, {1, -1}};
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) {
      const int kh = khs[a][i], kw = khs[b][j];
      if (kh < 0 || kw < 0) continue;
      const int n = t.pack.ntaps++;
      t.pack.kh[n] = kh; t.pack.kw[n] = kw;
      t.dh[n] = kh == 2 ? -1 : 0; t.dw[n] = kw == 2 ? -1 : 0;
    }
  return t;
}
// folded Upsample2D, output parity (a, b): the folded taps with negated offsets, gathered from the gradient's parity plane
inline TapSet taps_up2_neg(int a, int b) {
  TapSet t = taps_up2(a, b);
  t.pack.transpose = 1;
  for (int k = 0; k < 4; ++k) { t.dh[k] = (signed char)-t.dh[k]; t.dw[k] = (signed char)-t.dw[k]; }
  return t;
}

// K-segment over the first C channels of `src` (a PF8 tensor of img_planes 8-channel planes per image) with packed weights
// `wpack` and tap set `t`; no fused GroupNorm.  The launcher derives the halo from (dh, dw).
inline void set_seg(ConvSeg& s, const __nv_bfloat16* src, int img_planes, int C, int H, int W, const __nv_bfloat16* wpack,
                    const TapSet& t) {
  s.src = src;
  s.wpack = wpack;
  s.img_stride = (long long)img_planes * make_geom(1, H, W).PL * 8;
  s.ksteps = C / 16;
  s.ntaps = t.pack.ntaps;
  for (int k = 0; k < t.pack.ntaps; ++k) { s.dh[k] = t.dh[k]; s.dw[k] = t.dw[k]; }
  s.ss = nullptr; s.ss_stride = 0; s.silu = 0;
}

}  // namespace b200ad
