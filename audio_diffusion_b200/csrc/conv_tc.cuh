// Parameter block of the wgmma implicit-GEMM convolution (conv_tc.cu). Host + device.
#pragma once
#include "common.cuh"

namespace b200ad {

constexpr int CONV_NT = 128;        // output-channel tile = 2 x MMA M (one 64-row half per consumer warpgroup)
constexpr int CONV_TM = 128;        // pixels per tile; an MMA covers up to two tiles (N = 256)
constexpr int CONV_MAXG = 2;        // pixel tiles per work item: 64 x 256 fp32 accumulators = 128 registers per thread
constexpr int CONV_MAXSEG = 6;      // K-segments per launch (callers use up to 4; the launcher may split one, see below)
constexpr int CONV_MAXTAPS = 9;
constexpr int CONV_MAXSCHED = 256;  // k-steps of one item (all segments); a k-step index within its segment is 8 bits
constexpr int CONV_B_TAP = 16 * CONV_NT * 2;     // one tap, 16 input channels: 4096 B
constexpr int CONV_SMEM_MAX = 227 * 1024;

// Shared memory holds two independent rings: CONV_AS activation slots (one 16-channel k-step each: two 8-channel
// windows) and CONV_BS weight slots of CONV_BT taps each, so weights (the bulk of the bytes) are prefetched at a finer
// grain and the TMA -> transform -> MMA chain of the activations gets a deeper ring.
constexpr int CONV_BT = 3;                       // taps per weight slot
constexpr int CONV_B_SLOT = CONV_BT * CONV_B_TAP;
constexpr int CONV_AS_MAX = 8;    // launches with small windows use more activation stages (see launch_conv_tc)
constexpr int CONV_AS = 3;        // minimum activation-ring depth
constexpr int CONV_BS = 5;        // minimum weight-ring depth (W = 256: shared memory is full)
constexpr int CONV_BS_MAX = 10;   // launches with smaller activation stages use the rest for a deeper weight ring

// One K-segment: a source tensor (PF8) with its tap set and packed weights. A 3x3 conv is one
// segment with 9 taps; a fused 1x1 shortcut adds one 1-tap segment per shortcut source; a stride-2
// conv is four segments (one per input parity plane).
struct ConvSeg {
  const __nv_bfloat16* src;    // PF8 activations, same geometry as the output
  const __nv_bfloat16* wpack;  // [cout/128][ksteps][ntaps][2 k8][16 rows8][8][8] bf16, rows in channel order
  long long img_stride;        // elements between images of src (= C/8 * PL * 8)
  long long wtile_stride;      // elements between cout tiles of wpack (0: ksteps * ntaps * 2048; set by the launcher)
  int ksteps;                  // input channels / 16
  int ntaps;
  int ht, hb, hl, hr;          // halo rows above / below, pixels left / right
  signed char dh[CONV_MAXTAPS];
  signed char dw[CONV_MAXTAPS];
  int aoff[CONV_MAXTAPS];      // (dh + ht) * Wp + dw + hl, filled in by launch_conv_tc: window offset of each tap
  // Fused GroupNorm(+SiLU) of this source, applied to the A strips in shared memory before the MMAs read them:
  // value = silu?(x * ss[n][c].x + ss[n][c].y), forced to 0 on pad / guard positions. nullptr: source is used as is.
  const float2* ss;            // [N][ss_stride] (pointer already offset to this source's first channel)
  int ss_stride;
  int silu;
};

// GroupNorm statistics -> per-(sample, channel) (scale, shift) of the NEXT GroupNorm, computed by the last CTA of the
// launch that completes the statistics (no separate launch): `ss[n][c] = (gamma[c] * rstd, beta[c] - mean * gamma[c] * rstd)`
// over the channel concatenation of up to two tensors (the second one, a skip connection, was finished long before).
struct ConvGnFin {
  const stat_t* stats[2];   // [N][C_i / 4][2] quad (sum, sumsq)
  int C[2];
  const float* gamma;       // [C0 + C1]
  const float* beta;
  float2* ss;               // [N][C0 + C1]; nullptr: this launch finalises nothing
  unsigned* counter;        // CTA arrival counter (zero before and after every launch)
  int groups, HW;
  float eps;
};

struct ConvParams {
  ConvSeg seg[CONV_MAXSEG];
  int nseg;
  int N, H, W, Wp, lead, PL;
  int ktotal;           // sum of the segments' k-steps (set by the launcher)
  // Order of the k-steps of an item, (segment << 8) | k-step (set by the launcher): segment by segment.  Experiment
  // (B200AD_CONV_DBG & 2048): many-tap and 1-tap k-steps (shortcut, residual) interleaved, to spread the 1-tap k-steps'
  // window loads between many-tap k-steps.
  unsigned short sched[CONV_MAXSCHED];
  int a_stage;          // bytes reserved for the A strips of one stage (set by the launcher)
  int groups_per_img;
  int ntiles_n;         // cout / 128
  int total_work;       // N * groups_per_img * ntiles_n  (packed: ceil(N / 4) * ntiles_n)
  int pack;             // 0, or the images per item (1, 2, 4) for small images (image + bottom halo fit one 128-pixel tile):
                        // an item's tiles are consecutive images, so a weight fetch and an N = 256 MMA serve several samples
  int as, bs;           // activation stages / weight-ring slots of this launch (set by the launcher)
  int pdl;              // launched with programmatic stream serialization (set by the launcher)
  int cout;
  __nv_bfloat16* out;           // PF8, cout channels
  const float* bias;            // [cout]
  const float* temb;            // optional per-sample additive term [N][temb_stride] (offset applied)
  int temb_stride;
  stat_t* stats;                // optional [N][cout/4][2] running (sum, sumsq) of the stored output
  // Folded nearest-2x upsample: the item geometry (N, H, W, ...) is the LOW-res input; low-res pixel (h, w) is stored at
  // (2h + oy, 2w + ox) of the (2H, 2W) output tensor. One launch per output parity (oy, ox) with pre-summed 2x2 weights.
  int up2, oy, ox;
  ConvGnFin fin;
  int dbg;                      // B200AD_CONV_DBG bit flags (timing experiments only): 2 no stores, 4 CTAs out of phase, 8 no epilogue work, 32 no weight loads, 64 no transform, 128 reorder 1-tap segments before the last main k-step, 256 no small-image packing, 512 rings fixed at CONV_AS stages / CONV_BS slots, 1024 no programmatic dependent launch, 2048 interleave 1-tap k-steps between many-tap ones
};

cudaError_t launch_conv_tc(const ConvParams& p, int num_sms, cudaStream_t stream);

// Identity weight blocks (W[co][ci] = delta) in the packed layout: a residual add is one extra 1-tap K-segment over the
// raw source, accumulated by the tensor core (exact: bf16 * 1.0 into fp32).
cudaError_t launch_pack_identity(int channels, __nv_bfloat16* dst, cudaStream_t s);

}  // namespace b200ad
