// wgmma implicit-GEMM convolution for the U-Net hot path (replaces the cuDNN conv2d calls that
// diffusers' UNet2DModel.forward makes; reference call site audiodiffusion/pipeline_audio_diffusion.py:163).
//
// GEMM view (transposed): D^T[cout, pixel] = sum over (segment, tap, cin) W[cout, cin, tap] * X[pixel + shift(tap), cin].
//   M = 128 output channels (weights are the A operand; two consumer warpgroups take 64 rows each), N = up to 256 output
//   pixels (activations are the B operand), K = 16 input channels per wgmma.m64nNk16.  The accumulators of an item
//   (64 x 256 fp32 per warpgroup) live in registers, which caps an item at two 128-pixel tiles.
// Pixel operand: the PF8 layout stores 8-channel vectors of consecutive pixels contiguously, which *is* the K-major
//   no-swizzle core-matrix layout (8 rows x 16 B); along N the core matrices follow each other at a uniform stride (SBO).
//   A work item covers 256 output pixels in one of two shapes, chosen per launch from the shape alone:
//   - flat: 2 x 128 consecutive flat pixels.  Per 16 input channels ONE contiguous window per 8-channel plane (the run
//     plus a halo of Wp+1 pixels on both sides) is bulk-copied (TMA engine) into shared memory; SBO = 128 B and every tap
//     is a descriptor whose start address is shifted by (dh*Wp + dw) * 16 B.  (Few large copies: a bulk copy has a fixed
//     cost however small it is.)
//   - 2-D tile (ConvParams::tile2d): tw columns x th rows, 8 x 32 or 16 x 16.  Per 16 input channels one tensor-map copy
//     lands the box [2 planes][th + ht + hb rows][tw + hl + hr cols][8 ch]; each 8-column row of a tile is one core matrix,
//     so SBO is the box row pitch (tw + hl + hr) * 16 B and a tap shifts the start address by (dh * pitch + dw) * 16 B.
//     8 x 32 is one N = 256 MMA per tap; 16 x 16 is two 8-column halves of 16 rows, one N = 128 MMA each (the second
//     starts 8 pixels into the window), accumulating into the registers of flat tiles 0 and 1.  At W = 256 the window
//     is 10 x 34 pixels instead of 772, so each input pixel is loaded and normalised about once instead of three times;
//     at 16 x 16 and 32 x 32 an image is one or four whole items instead of 1.5 or 4.125 flat ones.  Elements outside
//     the image are zero-filled by the copy (the box is clipped at W, not at the pad column).
// Fused GroupNorm(+SiLU): the windows hold the RAW producer output; the transform warps rewrite them in place
//   (x * scale[n][c] + shift[n][c], SiLU via one tanh.approx, zero on pad/guard positions) between the TMA landing and
//   the MMA reading them, so the normalised tensor never exists in HBM.
// Weights: pre-packed on the device into per-(cout tile, 16-channel step, tap) 4 KB blocks; a separate, finer ring
//   (CONV_BT taps per slot) with its own producer warp.
// Residual adds are an extra 1-tap K-segment with identity weights (exact, and no epilogue loads).
// MMA pipeline: a consumer warpgroup issues the taps of one weight slot as one wgmma group and keeps one group in flight;
//   a weight slot (and, after the last slot of a k-step, the activation stage) is released once its group has retired.
// Epilogue (per consumer warpgroup, from registers): +bias/temb and GroupNorm partial sums -> cvt.rn.bf16x2 ->
//   stmatrix.trans into a staging buffer ([plane][pixel][8 ch] = finished PF8 runs; the wgmma fragment puts the 8 channels
//   of a plane in lanes 4 apart, which is exactly a transposed 8x8 matrix) -> bulk stores (TMA engine) draining while the
//   next item is multiplied.  Flat items: one bulk store per plane and tile; pad columns and the run-off behind the image
//   are stored as the zeros the layout requires there.  2-D tiles: the staging pixels of a 128-pixel half are
//   tile-row-major; 8 x 32: one tensor-map store writes the warpgroup's 8 planes, 16 x 16: one per (half, plane), like the
//   flat runs; every pixel is inside the image, so pads and guards are never written (they are zero from the workspace
//   memset at bind time and no writer of a PF8 tensor puts anything else there).  A folded upsample on 2-D tiles stores
//   through a map of its output parity (a strided view of the 2x tensor); on flat items it scatters from the staging rows.
// Small images (H * Wp + bottom halo <= 128 pixels: 8x8 and below): an item's tiles are the first tiles of CONSECUTIVE
//   IMAGES, so one weight fetch and one N = 256 MMA serve two samples (ConvParams::pack).
// Warp roles (12 warps): 0 activation producer, 1 weight producer, 2-3 transform, 4-7 and 8-11 the two consumer
//   warpgroups (MMA + epilogue).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <cstdlib>

#include "conv_tc.cuh"

namespace b200ad {

// Tensor maps of a 2-D-tiled launch (encoded by launch_conv_tc, see encode_pf8_map; unused by flat launches).  4-D over a
// PF8 tensor: {8 W elements (a row's pixels, 8 channels each), H rows, 8-channel planes, images}, based at pixel (0, 0) of
// plane 0.
struct alignas(64) ConvMaps {
  CUtensorMap src[CONV_MAXSEG];   // box {8 (tw + hl + hr), th + ht + hb, 2, 1}: one k-step's window of segment s
  CUtensorMap out;                // 8 x 32: box {64, 32, 8, 1}, a consumer warpgroup's staging buffer; 16 x 16: box
                                  // {64, 16, 1, 1}, one half-plane of it.  Folded upsample (16 x 16 only): 5-D over the
                                  // columns / rows of the output parity (stride 2 in the 2x tensor), box {8, 8, 16, 1, 1}
};

// pixels per 8-channel plane of a segment's window (G: the item's 128-pixel tiles, flat items only)
__host__ __device__ __forceinline__ int window_pixels(const ConvParams& p, const ConvSeg& sg, int G) {
  return p.tile2d ? (p.tw + sg.hl + sg.hr) * (p.th + sg.ht + sg.hb)
                  : G * CONV_TM + (sg.ht + sg.hb) * p.Wp + sg.hl + sg.hr;
}
// pixels from one window row to the next
__host__ __device__ __forceinline__ int window_pitch(const ConvParams& p, const ConvSeg& sg) {
  return p.tile2d ? p.tw + sg.hl + sg.hr : p.Wp;
}

constexpr int CONV_THREADS = 384;     // 12 warps
constexpr int CONV_XF_THREADS = 64;   // transform warps 2, 3
// epilogue staging, one buffer per consumer warpgroup: its 8 planes (64 channels) x 256 pixels, bf16
constexpr int CONV_SPLANE = CONV_MAXG * CONV_TM * 16;   // bytes per 8-channel plane of a buffer
constexpr int CONV_STG_WG = 8 * CONV_SPLANE;
constexpr int CONV_STAGING = 2 * CONV_STG_WG;
static size_t conv_smem_bytes(const ConvParams& p) {
  return (size_t)p.as * p.a_stage + (size_t)p.bs * CONV_B_SLOT + CONV_STAGING + 1024;
}

struct WorkItem {
  int n, ntile, m0, G;
  int r0, c0;   // 2-D tiles: first row / column of the tile
};

__device__ __forceinline__ WorkItem decode_work(const ConvParams& p, int w) {
  WorkItem wi;
  wi.ntile = w % p.ntiles_n;
  const int gidx = w / p.ntiles_n;
  if (p.tile2d) {   // tiles in column-major order: consecutive CTAs take vertically adjacent tiles, whose halos overlap in L2
    wi.n = gidx / p.groups_per_img;
    const int t = gidx - wi.n * p.groups_per_img, tx = t / p.tiles_y;
    wi.r0 = (t - tx * p.tiles_y) * p.th;
    wi.c0 = tx * p.tw;
    wi.m0 = 0;
    wi.G = CONV_MAXG;
    return wi;
  }
  wi.r0 = wi.c0 = 0;
  if (p.pack) {   // small images: the item's tiles are the first (only) tiles of p.pack (1, 2 or 4) CONSECUTIVE IMAGES n, n+1, ..
    wi.n = gidx * p.pack;
    wi.m0 = 0;
    wi.G = min(p.pack, p.N - wi.n);
    return wi;
  }
  wi.n = gidx / p.groups_per_img;
  const int g = gidx - wi.n * p.groups_per_img;
  wi.m0 = g * (CONV_MAXG * CONV_TM);
  const int rem = p.H * p.Wp - wi.m0;
  wi.G = min(CONV_MAXG, (rem + CONV_TM - 1) / CONV_TM);
  return wi;
}

// one 16-byte vector (8 channels of one pixel): affine + optional SiLU in fp32 (packed pairs), back to bf16.
// With SiLU the caller passes HALVED scale/shift: h = a/2 = x*s' + t', silu(a) = a * (0.5 + 0.5 tanh(a/2)) = h + h * tanh(h)
// -> per two elements: FFMA2, 2 MUFU.TANH, FFMA2.
template <bool SILU>
__device__ __forceinline__ uint4 xform_vec(uint4 v, const f32x2_t (&sc)[4], const f32x2_t (&sh)[4]) {
  uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    f32x2_t a = f2_fma(f2_from_bf16x2(u[e]), sc[e], sh[e]);
    if (SILU) {
      const float2 f = f2_unpack(a);
      a = f2_fma(a, f2_pack(tanh_approx(f.x), tanh_approx(f.y)), a);
    }
    u[e] = f2_to_bf16x2(a);
  }
  return make_uint4(u[0], u[1], u[2], u[3]);
}

// SQUARE: the launch's items are 16 x 16 tiles.  A separate instantiation: with the N = 256 MMA of the other shapes and
// the second N = 128 MMA (accumulators from acc[64]) in one function, ptxas serialises every wgmma (C7511).
template <bool SQUARE>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvParams p,
                                                                  const __grid_constant__ ConvMaps maps) {
  constexpr int ASM = CONV_AS_MAX, BSM = CONV_BS_MAX;
  const int AS = p.as;      // activation stages of this launch (CONV_AS .. CONV_AS_MAX)
  const int BS = p.bs;      // weight-ring depth of this launch (whatever the activation stages leave, CONV_BS .. CONV_BS_MAX)
  extern __shared__ __align__(128) uint8_t smem[];
  // Broadcast from lane 0 so that ptxas can prove the role branches warp-uniform; otherwise it treats the consumer's wgmma
  // loop as a divergent path and waits for every wgmma to complete before issuing the next (C7520).
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int a_bytes = p.a_stage;

  uint8_t* bring = smem + AS * a_bytes;                 // weight ring
  uint8_t* stg = bring + BS * CONV_B_SLOT;              // epilogue staging: one buffer per consumer warpgroup
  uint8_t* ctrl = stg + CONV_STAGING;
  // barriers: fullA[AS], readyA[AS], emptyA[AS], fullB[BS], emptyB[BS]
  uint64_t* bars = reinterpret_cast<uint64_t*>(ctrl);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bring_base = smem_u32(bring);
  const uint32_t bar_fullA = smem_u32(bars);
  const uint32_t bar_readyA = smem_u32(bars + ASM);
  const uint32_t bar_emptyA = smem_u32(bars + 2 * ASM);
  const uint32_t bar_fullB = smem_u32(bars + 3 * ASM);
  const uint32_t bar_emptyB = smem_u32(bars + 3 * ASM + BSM);
  static_assert((3 * ASM + 2 * BSM) * 8 <= 1024, "barrier block overflows");

  if (warp == 1 && lane == 0) {
    for (int s = 0; s < AS; ++s) {
      mbar_init(bar_fullA + 8 * s, 1);
      mbar_init(bar_readyA + 8 * s, CONV_XF_THREADS / 32);   // one arrival per transform warp
      mbar_init(bar_emptyA + 8 * s, 8);                       // one arrival per consumer warp
    }
    for (int s = 0; s < BS; ++s) {
      mbar_init(bar_fullB + 8 * s, 1);
      mbar_init(bar_emptyB + 8 * s, 8);
    }
    mbar_fence_init();
  }
  __syncthreads();

  // Programmatic dependent launch: this grid may have been started while the previous kernel of the stream was still
  // draining (its last wave, its last-CTA GroupNorm finalize).  Everything above, and the weight producer's prefetch below,
  // touches nothing that kernel writes (the packed weights are older); every other role waits for it here.  The next
  // launch is released at once - it parks at this same point.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (warp != 1) asm volatile("griddepcontrol.wait;" ::: "memory");

  // Every role walks the k-steps of an item in the same order: segment by segment, k-step by k-step.
  if (warp == 0) {
    // ================================ activation producer: per k-step two windows (one per 8-channel plane), lanes 0 / 1
    // (2-D tiles: one box holding both)
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
      const WorkItem wi = decode_work(p, w);
      for (int s = 0; s < p.nseg; ++s) {
        const ConvSeg& sg = p.seg[s];
        const uint32_t row_bytes = (uint32_t)window_pixels(p, sg, wi.G) * 16u;
        for (int ks = 0; ks < sg.ksteps; ++ks) {
          const uint32_t full = bar_fullA + 8 * stage;
          if (lane == 0) {
            mbar_wait(bar_emptyA + 8 * stage, phase ^ 1);
            mbar_arrive_expect_tx(full, 2u * row_bytes);
          }
          __syncwarp();
          const long long plane = (long long)(2 * ks + (lane & 1)) * p.PL;     // this lane's 8-channel plane of the k-step
          if (p.tile2d) {   // both planes in one box
            if (lane == 0)
              tensor_g2s_4d(smem_base + stage * a_bytes, &maps.src[s], 8 * (wi.c0 - sg.hl), wi.r0 - sg.ht, 2 * ks, wi.n, full);
          } else if (!p.pack) {
            const int pix0 = p.lead + wi.m0 - sg.ht * p.Wp - sg.hl;
            if (lane < 2)
              bulk_g2s(smem_base + stage * a_bytes + (uint32_t)lane * row_bytes,
                       sg.src + (long long)wi.n * sg.img_stride + (plane + pix0) * 8, row_bytes, full);
          } else {
            // packed small images: the window is [leading halo | tile 0 = image n | tile 1 = image n+1 | .. | trailing halo];
            // lane 2g + plane copies tile g (tile 0 with the leading halo, the last tile with the trailing one) of its plane.
            // Everything behind an image's H * Wp pixels is the zero guard of its own plane.
            const int g = lane >> 1, lead_px = sg.ht * p.Wp + sg.hl, trail_px = sg.hb * p.Wp + sg.hr;
            const int cnt = CONV_TM + (g == 0 ? lead_px : 0) + (g == wi.G - 1 ? trail_px : 0);
            const int doff = (g == 0) ? 0 : lead_px + g * CONV_TM;                      // pixels into the plane's window
            const int pix0 = p.lead - (g == 0 ? lead_px : 0);
            if (g < wi.G && lane < 2 * CONV_MAXG)
              bulk_g2s(smem_base + stage * a_bytes + (uint32_t)(lane & 1) * row_bytes + (uint32_t)doff * 16u,
                       sg.src + (long long)(wi.n + g) * sg.img_stride + (plane + pix0) * 8, (uint32_t)cnt * 16u, full);
          }
          if (++stage == AS) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp == 1) {
    // ================================ weight producer: slots of up to CONV_BT taps (12 KB), one bulk copy each
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
        const int ntile = w % p.ntiles_n;
        for (int s = 0; s < p.nseg; ++s) {
          const ConvSeg& sg = p.seg[s];
          // a segment's weights of one cout tile are its k-steps' tap blocks, one after the other
          const char* src = reinterpret_cast<const char*>(sg.wpack + (long long)ntile * sg.wtile_stride);
          for (int ks = 0; ks < sg.ksteps; ++ks) {
            for (int t0 = 0; t0 < sg.ntaps; t0 += CONV_BT) {
              const uint32_t bytes = (uint32_t)min(CONV_BT, sg.ntaps - t0) * CONV_B_TAP;
              mbar_wait(bar_emptyB + 8 * stage, phase ^ 1);
              if (p.dbg & 32) {      // experiment: no weight traffic at all (bounds what sharing weight fetches could buy)
                mbar_arrive(bar_fullB + 8 * stage);
              } else {
                mbar_arrive_expect_tx(bar_fullB + 8 * stage, bytes);
                bulk_g2s(bring_base + stage * CONV_B_SLOT, src, bytes, bar_fullB + 8 * stage);
              }
              src += bytes;
              if (++stage == BS) { stage = 0; phase ^= 1; }
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ================================ consumer warpgroup cw: output channels [64 cw, 64 cw + 64) of the item's cout tile.
    // Accumulator fragment: warp wq, lane l holds channels 64 cw + 16 wq + l/4 (h = 0) and +8 (h = 1) for pixels
    // 8j + 2 (l % 4) + {0, 1} in acc[4j + 2h + {0, 1}].
    const int cw = (warp - 4) >> 2, wq = warp & 3, tid = threadIdx.x & 127;
    const uint32_t stg_w = smem_u32(stg) + (uint32_t)(cw * CONV_STG_WG);
    // stmatrix.x4.trans row address of this lane: matrix m = lane >> 3 is (8-pixel group 2k + (m >> 1), plane 2 wq + (m & 1)),
    // row r = lane & 7 is pixel r of that group; element c of the row comes from lane 4c + r / 2
    const uint32_t st_addr = stg_w + (uint32_t)((2 * wq + ((lane >> 3) & 1)) * CONV_SPLANE + (8 * (lane >> 4) + (lane & 7)) * 16);
    const Geom og = make_geom(p.N, p.up2 ? 2 * p.H : p.H, p.up2 ? 2 * p.W : p.W);   // geometry of the output tensor
    const long long out_img_stride = (long long)(p.cout >> 3) * og.PL * 8;
    const int hw_end = p.H * p.Wp;
    const bool do_stats = p.stats != nullptr;
    const bool issuer = tid < 8 * CONV_MAXG;   // thread (tile g, plane pl) = (tid >> 3, tid & 7) bulk-stores one run
    float acc[CONV_MAXG * CONV_TM / 2];
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
      const WorkItem wi = decode_work(p, w);
#pragma unroll
      for (int i = 0; i < CONV_MAXG * CONV_TM / 2; ++i) acc[i] = 0.f;
      // MMA groups: one per weight slot, one group in flight; pend_* = the slots of the group before the current one
      int pend_b = -1, pend_a = -1;
      auto release = [&]() {
        __syncwarp();
        if (lane == 0) {
          if (pend_b >= 0) mbar_arrive(bar_emptyB + 8 * pend_b);
          if (pend_a >= 0) mbar_arrive(bar_emptyA + 8 * pend_a);
        }
      };
      // one loop with a (segment, k-step) cursor: nested loops cost this role two registers (162 instead of 160)
      for (int s = 0, ks = 0; s < p.nseg;) {
        const ConvSeg& sg = p.seg[s];
        const uint32_t xlbo = (uint32_t)window_pixels(p, sg, wi.G) * 16u;   // the second 8-channel plane of the window
        const uint32_t xsbo = p.tile2d ? (uint32_t)window_pitch(p, sg) * 16u : 128u;   // the next 8 pixels along N
        const int ntaps = sg.ntaps;
        mbar_wait(bar_readyA + 8 * sa, pa);   // windows landed and (if asked) normalised in place
        const uint32_t abase = smem_base + sa * a_bytes;
        for (int t0 = 0; t0 < ntaps; t0 += CONV_BT) {
          mbar_wait(bar_fullB + 8 * sb, pb);  // this slot's taps landed
          const uint32_t bbase = bring_base + sb * CONV_B_SLOT + (uint32_t)(cw * 1024);   // rows 64 cw .. 64 cw + 63
          const int nt = min(CONV_BT, ntaps - t0);
          wgmma_fence();
          for (int t = 0; t < nt; ++t) {
            const uint64_t wdesc = gmma_desc(bbase + (uint32_t)t * CONV_B_TAP, (CONV_NT / 8) * 128, 128);
            const uint64_t xdesc = gmma_desc(abase + (uint32_t)sg.aoff[t0 + t] * 16u, xlbo, xsbo);
            if constexpr (SQUARE) {   // columns 0-7 into acc[0..63], columns 8-15 (8 pixels = 128 B on) into acc[64..127]
              wgmma_m64n128k16_x2(acc, wdesc, xdesc, xdesc + (128u >> 4));
            } else if (wi.G == 2) {
              wgmma_m64n256k16<0, 0>(acc, wdesc, xdesc);
            } else {
              wgmma_m64n128k16<0, 0>(acc, wdesc, xdesc);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous group has retired: its slots are free
          release();
          pend_b = sb;
          pend_a = (t0 + CONV_BT >= ntaps) ? sa : -1;
          if (++sb == BS) { sb = 0; pb ^= 1; }
        }
        if (++sa == AS) { sa = 0; pa ^= 1; }
        if (++ks == sg.ksteps) { ks = 0; ++s; }
      }
      wgmma_wait<0>();
      release();

      // ---- epilogue. The staging buffer is free once this warpgroup's bulk stores of the previous item have read it.
      if (issuer) bulk_wait_read_all();
      named_bar_sync(1 + cw, 128);
      if (!(p.dbg & 8)) {
        float ssum[2] = {0.f, 0.f}, ssq[2] = {0.f, 0.f};   // partial sums of this thread's two channels
#pragma unroll
        for (int g = 0; g < CONV_MAXG; ++g) {
          if (g < wi.G) {
            const int n = p.pack ? wi.n + g : wi.n;
            float bias[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int c = wi.ntile * CONV_NT + cw * 64 + wq * 16 + 8 * h + (lane >> 2);
              bias[h] = p.bias ? __ldg(p.bias + c) : 0.f;
              if (p.temb) bias[h] += __ldg(p.temb + (long long)n * p.temb_stride + c);
            }
            // first pixel of this thread within its image, and its column
            int m = (p.pack ? 0 : wi.m0 + g * CONV_TM) + 2 * (lane & 3);
            int col = m % p.Wp;
#pragma unroll
            for (int k = 0; k < CONV_TM / 16; ++k) {   // two 8-pixel groups per stmatrix.x4
              uint32_t pk[4];
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                // pad columns and the run-off behind the image are written as ZEROS (they are zero guards of the layout)
                // and do not count for the statistics (a 2-D tile has none)
                const int col1 = (col + 1 == p.Wp) ? 0 : col + 1;
                const bool v0 = p.tile2d || (m < hw_end && col < p.W), v1 = p.tile2d || (m + 1 < hw_end && col1 < p.W);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int j = g * (CONV_TM / 8) + 2 * k + u;
                  const float a0 = v0 ? acc[4 * j + 2 * h] + bias[h] : 0.f;
                  const float a1 = v1 ? acc[4 * j + 2 * h + 1] + bias[h] : 0.f;
                  ssum[h] += a0 + a1;
                  ssq[h] = fmaf(a0, a0, fmaf(a1, a1, ssq[h]));
                  pk[2 * u + h] = pack_bf16x2(a0, a1);
                }
                m += 8;
                col += 8;
                while (col >= p.Wp) col -= p.Wp;
              }
              stmatrix_x4_trans(st_addr + (uint32_t)((g * CONV_TM + 16 * k) * 16), pk[0], pk[1], pk[2], pk[3]);
            }
            if (do_stats && (p.pack || g == wi.G - 1)) {
              // quad (4-channel) sums: the 4 lanes of a channel and the 4 channels of a quad are the lanes of a half-warp
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float s1 = ssum[h], s2 = ssq[h];
#pragma unroll
                for (int o = 1; o < 16; o <<= 1) {
                  s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                  s2 += __shfl_xor_sync(0xffffffffu, s2, o);
                }
                if ((lane & 15) == 0) {
                  const int c = wi.ntile * CONV_NT + cw * 64 + wq * 16 + 8 * h + (lane >> 2);
                  stat_t* sdst = p.stats + ((long long)n * (p.cout >> 2) + (c >> 2)) * 2;
                  atomicAdd(sdst, (stat_t)s1);
                  atomicAdd(sdst + 1, (stat_t)s2);
                }
                ssum[h] = 0.f;
                ssq[h] = 0.f;
              }
            }
          }
        }
      }
      if (p.tile2d) {
        fence_proxy_async_smem();   // staging rows written through the generic proxy -> visible to the TMA engine
        named_bar_sync(1 + cw, 128);
        if (SQUARE) {               // thread (half g, plane pl) = (tid >> 3, tid & 7) stores one 8 x 16 half-plane
          const int g = tid >> 3, pl = tid & 7;
          if (issuer && !(p.dbg & 2)) {
            const uint32_t src = stg_w + (uint32_t)(pl * CONV_SPLANE + g * CONV_TM * 16);
            const int c = wi.c0 + 8 * g, plane = wi.ntile * 16 + cw * 8 + pl;
            if (p.up2) tensor_s2g_5d(&maps.out, 0, c, wi.r0, plane, wi.n, src);
            else       tensor_s2g_4d(&maps.out, 8 * c, wi.r0, plane, wi.n, src);
            bulk_commit();
          }
        } else if (tid == 0 && !(p.dbg & 2)) {
          tensor_s2g_4d(&maps.out, 8 * wi.c0, wi.r0, wi.ntile * 16 + cw * 8, wi.n, stg_w);   // never an upsample
          bulk_commit();
        }
      } else if (!p.up2) {
        fence_proxy_async_smem();
        named_bar_sync(1 + cw, 128);
        const int g = tid >> 3, pl = tid & 7;
        if (issuer && g < wi.G && !(p.dbg & 2)) {
          const int n = p.pack ? wi.n + g : wi.n;
          bulk_s2g(p.out + (long long)n * out_img_stride + (long long)(wi.ntile * 16 + cw * 8 + pl) * og.PL * 8 +
                       (long long)(p.lead + (p.pack ? 0 : wi.m0 + CONV_TM * g)) * 8,
                   stg_w + (uint32_t)(pl * CONV_SPLANE + g * CONV_TM * 16), (uint32_t)CONV_TM * 16u);
          bulk_commit();
        }
      } else {
        // folded upsample on flat items: scatter into the 2x tensor at this launch's parity, straight from the staging rows
        named_bar_sync(1 + cw, 128);
        const int npx = wi.G * CONV_TM;
        for (int i = tid; i < 8 * npx && !(p.dbg & 2); i += 128) {
          const int pl = i / npx, px = i - pl * npx, g = px >> 7;
          const int m = p.pack ? px & (CONV_TM - 1) : wi.m0 + px;
          const int hh = m / p.Wp, ww = m - hh * p.Wp;
          if (m < hw_end && ww < p.W) {
            const int n = p.pack ? wi.n + g : wi.n;
            const uint4 o = *reinterpret_cast<const uint4*>(stg + cw * CONV_STG_WG + pl * CONV_SPLANE + px * 16);
            *reinterpret_cast<uint4*>(p.out + (long long)n * out_img_stride + (long long)(wi.ntile * 16 + cw * 8 + pl) * og.PL * 8 +
                                      (long long)(og.lead + (2 * hh + p.oy) * og.Wp + 2 * ww + p.ox) * 8) = o;
          }
        }
      }
    }
    if (issuer) bulk_wait_all();   // shared memory must outlive the engine's reads; the stores complete before the CTA exits
  } else {
    // ================================ transform warps (2, 3): GroupNorm(+SiLU) of the landed windows, in place.
    // Every 64-pixel sweep of a window is two groups of 32 pixels, one per transform warp.
    const int tidx = (warp - 2) * 32 + lane;   // this thread's first pixel of a window
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
      const WorkItem wi = decode_work(p, w);
      for (int s = 0; s < p.nseg; ++s) {
        const ConvSeg& sg = p.seg[s];
        const int npix = window_pixels(p, sg, wi.G);
        const int pitch = window_pitch(p, sg);
        const float2* ssn = sg.ss ? sg.ss + (long long)wi.n * sg.ss_stride : nullptr;
        // Window pixel i is image pixel (row, cbase + col), col in [0, pitch): flat items start at flat position
        // m0 - ht * Wp - hl (cbase 0), 2-D tiles at (r0 - ht, c0 - hl).  (row, col) of this thread's pixel advance
        // incrementally (one sweep per iteration).
        const int cbase = p.tile2d ? wi.c0 - sg.hl : 0;
        int row0, col0;
        if (p.tile2d) {
          row0 = wi.r0 - sg.ht + tidx / pitch;
          col0 = tidx - (tidx / pitch) * pitch;
        } else {
          const int m_first = wi.m0 - sg.ht * p.Wp - sg.hl + tidx;
          row0 = (m_first >= 0) ? m_first / p.Wp : -1 - ((-1 - m_first) / p.Wp);  // floor division
          col0 = m_first - row0 * p.Wp;
        }
        const int drow = CONV_XF_THREADS / pitch;
        const int dcol = CONV_XF_THREADS - drow * pitch;
        const bool silu = sg.silu != 0;
        for (int ks = 0; ks < sg.ksteps; ++ks) {
          f32x2_t sc0[4], sh0[4], sc1[4], sh1[4];
          if (ssn && !p.pack) {
            const float4* sp = reinterpret_cast<const float4*>(ssn + ks * 16);
            const float hs = silu ? 0.5f : 1.0f;  // SiLU path works on a/2 (see xform_vec)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float4 a = __ldg(sp + e), b = __ldg(sp + 4 + e);   // (scale, shift) of channels 2e, 2e+1 | 8+2e, 9+2e
              sc0[e] = f2_pack(a.x * hs, a.z * hs); sh0[e] = f2_pack(a.y * hs, a.w * hs);
              sc1[e] = f2_pack(b.x * hs, b.z * hs); sh1[e] = f2_pack(b.y * hs, b.w * hs);
            }
          }
          mbar_wait(bar_fullA + 8 * stage, phase);
          if (ssn && p.pack && !(p.dbg & 64)) {
            // packed small images: tile g holds image n + g (its own scale / shift); only the image's valid pixels are
            // touched - everything else in the window is zero guard from global memory and stays zero
            uint4* base = reinterpret_cast<uint4*>(smem + stage * a_bytes);
            const int lead_px = sg.ht * p.Wp + sg.hl, hw = p.H * p.Wp;
            const float hs = silu ? 0.5f : 1.0f;
            for (int g = 0; g < wi.G; ++g) {
              const float4* sp = reinterpret_cast<const float4*>(ssn + (long long)g * sg.ss_stride + ks * 16);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float4 a = __ldg(sp + e), b = __ldg(sp + 4 + e);
                sc0[e] = f2_pack(a.x * hs, a.z * hs); sh0[e] = f2_pack(a.y * hs, a.w * hs);
                sc1[e] = f2_pack(b.x * hs, b.z * hs); sh1[e] = f2_pack(b.y * hs, b.w * hs);
              }
              for (int m = tidx; m < hw; m += CONV_XF_THREADS) {
                const int r = m / p.Wp;
                const int px = lead_px + g * CONV_TM + m;
                uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);    // pad column: stays zero
                if (m - r * p.Wp < p.W) {
                  a = base[px];
                  b = base[npix + px];
                  if (silu) { a = xform_vec<true>(a, sc0, sh0); b = xform_vec<true>(b, sc1, sh1); }
                  else      { a = xform_vec<false>(a, sc0, sh0); b = xform_vec<false>(b, sc1, sh1); }
                }
                base[px] = a;
                base[npix + px] = b;
              }
            }
            fence_proxy_async_smem();
          } else if (ssn && !(p.dbg & 64)) {
            uint4* base = reinterpret_cast<uint4*>(smem + stage * a_bytes);
            int row = row0, col = col0;
            for (int px = tidx; px < npix; px += CONV_XF_THREADS) {
              const bool valid = (row >= 0) && (row < p.H) && ((unsigned)(cbase + col) < (unsigned)p.W);
              uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
              if (valid) {
                a = base[px];
                b = base[npix + px];
                if (silu) { a = xform_vec<true>(a, sc0, sh0); b = xform_vec<true>(b, sc1, sh1); }
                else      { a = xform_vec<false>(a, sc0, sh0); b = xform_vec<false>(b, sc1, sh1); }
              }
              base[px] = a;
              base[npix + px] = b;
              row += drow; col += dcol;
              if (col >= pitch) { col -= pitch; ++row; }
            }
            fence_proxy_async_smem();
          }
          // every lane has fenced its own writes towards the async proxy; the warp then arrives ONCE (32 same-address
          // shared-memory atomics per warp and k-step were ~7 % of the kernel's shared-memory wavefronts)
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_readyA + 8 * stage);
          if (++stage == AS) { stage = 0; phase ^= 1; }
        }
      }
    }
  }

  if (p.fin.ss) __threadfence();   // this thread's statistics atomics are ordered before the CTA's arrival below
  __syncthreads();

  // ---- GroupNorm finalize of the consumer, by the last CTA to arrive (replaces a launch per GroupNorm)
  if (p.fin.ss) {
    __shared__ unsigned s_last;
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = (atomicAdd(p.fin.counter, 1u) == gridDim.x - 1) ? 1u : 0u;
    }
    __syncthreads();
    if (s_last) {
      __threadfence();
      const ConvGnFin& f = p.fin;
      const int Ct = f.C[0] + f.C[1], cpg = Ct / f.groups;
      float* gmean = reinterpret_cast<float*>(smem);        // the rings are idle now: [N * groups] mean, then rstd
      float* grstd = gmean + p.N * f.groups;
      const double cnt = (double)cpg * (double)f.HW;
      // This tail runs on ONE CTA after the grid has drained, so its latency is exposed in every launch (about 15 us before
      // it was restructured, x 71 GroupNorms per step): the quad sums of a group are fetched as one batch of independent
      // 16-byte L2 loads (up to 8 in flight per thread) instead of a dependent chain, and the second pass walks (n, c)
      // incrementally (no integer divisions) with the affine parameters in registers.
      for (int i = threadIdx.x; i < p.N * f.groups; i += CONV_THREADS) {
        const int n = i / f.groups, gi = i - n * f.groups;
        double sm = 0., sq = 0.;
        for (int c0 = gi * cpg; c0 < (gi + 1) * cpg; c0 += 32) {
          double2 v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const int c = c0 + 4 * k;
            v[k] = make_double2(0., 0.);
            if (c < (gi + 1) * cpg) {
              const stat_t* st = (c < f.C[0]) ? f.stats[0] + ((long long)n * (f.C[0] >> 2) + (c >> 2)) * 2
                                              : f.stats[1] + ((long long)n * (f.C[1] >> 2) + ((c - f.C[0]) >> 2)) * 2;
              v[k] = __ldcg(reinterpret_cast<const double2*>(st));
            }
          }
#pragma unroll
          for (int k = 0; k < 8; ++k) { sm += v[k].x; sq += v[k].y; }
        }
        const double mean = sm / cnt;
        gmean[i] = (float)mean;
        grstd[i] = (float)(1.0 / sqrt(fmax(sq / cnt - mean * mean, 0.) + (double)f.eps));
      }
      __syncthreads();
      {
        const int total = p.N * Ct;
        const int dn = CONV_THREADS / Ct, dc = CONV_THREADS - dn * Ct;
        const float inv_cpg = 1.0f / (float)cpg;
        int i = threadIdx.x;
        int n = i / Ct, c = i - n * Ct;
        for (; i < total; i += CONV_THREADS) {
          const int gi = n * f.groups + (int)(((float)c + 0.5f) * inv_cpg);    // c / cpg (exact for these small integers)
          const float sc = __ldg(f.gamma + c) * grstd[gi];
          f.ss[i] = make_float2(sc, __ldg(f.beta + c) - gmean[gi] * sc);
          n += dn;
          c += dc;
          if (c >= Ct) { c -= Ct; ++n; }
        }
      }
      if (threadIdx.x == 0) *f.counter = 0u;
    }
  }
}

// Tensor map over `planes` 8-channel planes of a PF8 tensor: W x H pixels from pixel (0, 0) at `base`, `cs` / `rs` pixels
// apart along a row / a column, planes `pl` pixels apart, images `img_stride` elements apart.
// - cs == 1 (pixels of a row are contiguous): 4-D {8 W elements, H rows, planes, images}, box {8 bw, bh, bplanes, 1};
//   coordinates (8 * column, row, plane, image).  A box row is then ONE run of 8 bw elements (128 - 288 B) for the TMA
//   engine instead of bw separate 16-byte pixels, which it moves at a fraction of the rate.  Columns outside the image
//   read as zeros and are not written, as whole pixels.
// - otherwise (a folded upsample's output parity): 5-D {8, W, H, planes, images}, box {8, bw, bh, bplanes, 1};
//   coordinates (0, column, row, plane, image).
// The driver's encoder is reached through the runtime, so the library links only cudart.
static cudaError_t encode_pf8_map(CUtensorMap* m, const __nv_bfloat16* base, const ConvParams& p, int cs, int rs, long long pl,
                                  int planes, long long img_stride, int bw, int bh, int bplanes) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q);
    if (e != cudaSuccess) return e;
    if (q != cudaDriverEntryPointSuccess || !fn) return cudaErrorNotSupported;
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint32_t estride[5] = {1, 1, 1, 1, 1};
  CUresult r;
  if (cs == 1) {
    const cuuint64_t dim[4] = {(cuuint64_t)p.W * 8, (cuuint64_t)p.H, (cuuint64_t)planes, (cuuint64_t)p.N};
    const cuuint64_t stride[3] = {(cuuint64_t)rs * 16, (cuuint64_t)pl * 16, (cuuint64_t)img_stride * 2};
    const cuuint32_t box[4] = {(cuuint32_t)bw * 8, (cuuint32_t)bh, (cuuint32_t)bplanes, 1};
    r = encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)base, dim, stride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t dim[5] = {8, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)planes, (cuuint64_t)p.N};
    const cuuint64_t stride[4] = {(cuuint64_t)cs * 16, (cuuint64_t)rs * 16, (cuuint64_t)pl * 16, (cuuint64_t)img_stride * 2};
    const cuuint32_t box[5] = {8, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bplanes, 1};
    r = encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)base, dim, stride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

int conv_dbg_env() {
  // timing experiments only; read on every launch so that one process can alternate settings (tools/ab_conv.py)
  const char* dbg_env = getenv("B200AD_CONV_DBG");
  return dbg_env ? atoi(dbg_env) : 0;
}

cudaError_t plan_conv_tc(ConvParams& p, int num_sms) {
  if (p.nseg < 1 || p.nseg > CONV_MAXSEG) return cudaErrorInvalidValue;
  for (int s = 0; s < p.nseg; ++s) {
    ConvSeg& sg = p.seg[s];
    if (sg.ntaps > CONV_MAXTAPS || sg.ksteps < 1) return cudaErrorInvalidValue;
    if (sg.wtile_stride == 0) sg.wtile_stride = (long long)sg.ksteps * sg.ntaps * (CONV_B_TAP / 2);
    sg.ht = sg.hb = sg.hl = sg.hr = 0;
    for (int t = 0; t < sg.ntaps; ++t) {
      sg.ht |= sg.dh[t] < 0; sg.hb |= sg.dh[t] > 0;
      sg.hl |= sg.dw[t] < 0; sg.hr |= sg.dw[t] > 0;
    }
  }
  p.tile2d = 0;
  p.tw = p.th = 0;
  p.tiles_y = 0;
  p.groups_per_img = (p.H * p.Wp + CONV_MAXG * CONV_TM - 1) / (CONV_MAXG * CONV_TM);
  p.ntiles_n = p.cout / CONV_NT;
  p.total_work = p.N * p.groups_per_img * p.ntiles_n;
  // Small images (8x8 and below at the bottom of the U-Net, every level of the latent model below 16x16): one image is a
  // fraction of a tile, so an item per image fetches the full weight set (1.2 MB for 512 -> 512) for <= 72 pixels and runs
  // N = 128 MMAs.  Packed, an item holds the first tile of up to four consecutive images: the window of tile g is image
  // n + g's plane from its pixel 0 on, whose tail is that image's own zero guard, so every tap of a valid output pixel stays
  // inside its tile (needs H * Wp + the bottom halo <= 128) and the MMA issue is unchanged.
  p.pack = 0;
  int fits = 1;
  for (int s = 0; s < p.nseg; ++s) {
    const ConvSeg& sg = p.seg[s];
    if (p.H * p.Wp + sg.hb * p.Wp + sg.hr > CONV_TM || sg.ht * p.Wp + sg.hl > CONV_TM) fits = 0;
  }
  if (fits) {
    // images per item: the MMA time of an item grows with its tiles (1 : 2 : 4), the number of waves shrinks with them;
    // take the fewest (waves x tiles), the larger group on a tie (fewer weight fetches)
    int best = 1;
    long long best_cost = -1;
    for (int g = 1; g <= CONV_MAXG; g *= 2) {
      const long long items = (long long)((p.N + g - 1) / g) * p.ntiles_n;
      const long long cost = ((items + num_sms - 1) / num_sms) * g;
      if (best_cost < 0 || cost <= best_cost) { best_cost = cost; best = g; }
    }
    p.pack = best;
    p.total_work = ((p.N + best - 1) / best) * p.ntiles_n;
  }
  const int tiles_img = (p.H * p.Wp + CONV_TM - 1) / CONV_TM;
  const int max_g = p.pack ? p.pack : (tiles_img < CONV_MAXG ? tiles_img : CONV_MAXG);   // most tiles any item of this launch has
  // Item shape by cost per image and cout tile, compared in this order: MMA columns issued (a flat item whose second tile
  // would be empty runs N = 128), items (each streams the cout tile's whole weight set from L2), window bytes loaded and
  // normalised.  Flat items pay a halo of two image rows and, where H * Wp is not a multiple of 256, a part-empty last
  // item (16 x 16: 1.5 items per image, 32 x 32: 4.125); a 2-D tile covers whole image rows and columns.  Packed small
  // images are one tile each and stay flat.  Two exceptions, both measured (H100 80GB HBM3, 700 W, batch 64 at 256 x 256):
  // - 16 x 16 and 8 x 32 tie on the first two wherever both fit, and 16 x 16's window is 5 % smaller; images of 64 rows
  //   and more keep 8 x 32 (one N = 256 MMA per tap reads the weights from shared memory once, 16 x 16's two N = 128
  //   MMAs twice; 16 x 16 there cost about 0.7 ms more per denoising step).
  // - A folded upsample takes 16 x 16 tiles but not 8 x 32: its tile store through the parity map writes 16-byte pixels
  //   32 bytes apart, and at 128 -> 256 that took 0.9 ms per step more than the flat items' scatter.
  if (!p.pack && !(p.dbg & 4096)) {
    auto window_cost = [&](const ConvParams& q, int G) {
      long long c = 0;
      for (int s = 0; s < q.nseg; ++s) c += (long long)window_pixels(q, q.seg[s], G) * q.seg[s].ksteps;
      return c;
    };
    long long best[3] = {(long long)tiles_img * CONV_TM, p.groups_per_img, 0};
    for (int i = 0; i < p.groups_per_img; ++i) best[2] += window_cost(p, min(CONV_MAXG, tiles_img - CONV_MAXG * i));
    const int shapes[2][2] = {{8, 32}, {16, 16}};
    for (const auto& sh : shapes) {
      const int tw = sh[0], th = sh[1];
      if (p.W % tw || p.H % th) continue;
      if (tw == 16 && p.H >= 64 && p.H % 32 == 0 && p.W % 8 == 0) continue;
      if (tw == 8 && p.up2) continue;
      ConvParams q = p;
      q.tile2d = 1; q.tw = tw; q.th = th;
      const long long items = (long long)(p.W / tw) * (p.H / th);
      const long long c[3] = {items * CONV_MAXG * CONV_TM, items, items * window_cost(q, CONV_MAXG)};
      if (c[0] < best[0] || (c[0] == best[0] && (c[1] < best[1] || (c[1] == best[1] && c[2] < best[2])))) {
        best[0] = c[0]; best[1] = c[1]; best[2] = c[2];
        p.tile2d = 1; p.tw = tw; p.th = th;
      }
    }
    if (p.tile2d) {
      p.tiles_y = p.H / p.th;
      p.groups_per_img = (p.W / p.tw) * p.tiles_y;
      p.total_work = p.N * p.groups_per_img * p.ntiles_n;
    }
  }
  // the two windows of one k-step must fit an activation slot
  int a_stage = 0;
  for (int s = 0; s < p.nseg; ++s) {
    const ConvSeg& sg = p.seg[s];
    const int npix = window_pixels(p, sg, max_g), pitch = window_pitch(p, sg);
    a_stage = npix * 32 > a_stage ? npix * 32 : a_stage;
    if (sg.ntaps > CONV_MAXTAPS || sg.ntaps > CONV_BT * (CONV_BS - 1) || npix > 0x3FFF) return cudaErrorInvalidValue;
    for (int t = 0; t < sg.ntaps; ++t) p.seg[s].aoff[t] = (sg.dh[t] + sg.ht) * pitch + sg.dw[t] + sg.hl;
  }
  p.a_stage = (a_stage + 255) & ~255;
  // Ring depths: W = 256 fills shared memory with 3 activation stages + 5 weight slots.  Launches with smaller windows (narrow
  // images, packed small images, 1-tap convs) have SHORT k-steps, and the TMA -> transform -> MMA chain of a stage (a few
  // thousand cycles of L2 latency) is then covered only by more stages in flight: first up to 6 activation stages, then the
  // weight ring up to its maximum, then the remaining activation stages.
  p.as = CONV_AS;
  p.bs = CONV_BS;
  auto rings_fit = [&](int as, int bs) {
    // 1 KB of head room: the kernel's static shared memory counts against the same 227 KB
    return (size_t)as * p.a_stage + (size_t)bs * CONV_B_SLOT + CONV_STAGING + 2048 <= (size_t)CONV_SMEM_MAX;
  };
  while (p.as < 6 && rings_fit(p.as + 1, p.bs)) ++p.as;
  while (p.bs < CONV_BS_MAX && rings_fit(p.as, p.bs + 1)) ++p.bs;
  while (p.as < CONV_AS_MAX && rings_fit(p.as + 1, p.bs)) ++p.as;
  if (conv_smem_bytes(p) > (size_t)CONV_SMEM_MAX) return cudaErrorInvalidValue;  // image too wide for this tiling
  return cudaSuccess;
}

cudaError_t launch_conv_tc(const ConvParams& p_in, int num_sms, cudaStream_t stream) {
  ConvParams p = p_in;
  p.dbg = conv_dbg_env();
  if (cudaError_t e = plan_conv_tc(p, num_sms)) return e;
  ConvMaps maps{};
  if (p.tile2d) {
    for (int s = 0; s < p.nseg; ++s) {
      const ConvSeg& sg = p.seg[s];
      cudaError_t e = encode_pf8_map(&maps.src[s], sg.src + (long long)p.lead * 8, p, 1, p.Wp, p.PL, 2 * sg.ksteps,
                                     sg.img_stride, p.tw + sg.hl + sg.hr, p.th + sg.ht + sg.hb, 2);
      if (e != cudaSuccess) return e;
    }
    // 8 x 32: the warpgroup's 8 planes in one box; 16 x 16: one half-plane (8 columns x 16 rows) per box
    const int bh = p.th, bplanes = p.tw == 16 ? 1 : 8;
    cudaError_t e;
    if (p.up2) {   // low-res pixel (h, w) -> (2h + oy, 2w + ox) of the 2x tensor: every second column and row
      const Geom og = make_geom(p.N, 2 * p.H, 2 * p.W);
      e = encode_pf8_map(&maps.out, p.out + (long long)(og.lead + p.oy * og.Wp + p.ox) * 8, p, 2, 2 * og.Wp, og.PL,
                         p.cout / 8, (long long)(p.cout / 8) * og.PL * 8, 8, bh, bplanes);
    } else {
      e = encode_pf8_map(&maps.out, p.out + (long long)p.lead * 8, p, 1, p.Wp, p.PL, p.cout / 8,
                         (long long)(p.cout / 8) * p.PL * 8, 8, bh, bplanes);
    }
    if (e != cudaSuccess) return e;
  }
  const size_t smem = conv_smem_bytes(p);
  const int grid = p.total_work < num_sms ? p.total_work : num_sms;
  if (grid <= 0) return cudaSuccess;
  const bool square = p.tile2d && p.tw == 16;
  void (*kernel)(ConvParams, ConvMaps) = square ? conv_tc_kernel<true> : conv_tc_kernel<false>;
  static size_t attr[2] = {0, 0};
  if (smem > attr[square]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr[square] = smem;
  }
  // launch with programmatic stream serialization: the grid may begin (prologue, weight prefetch) before its predecessor
  // has completed; it synchronises on the predecessor itself (griddepcontrol.wait) before touching anything it depends on
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(CONV_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, p, maps);
}

// ------------------------------------------------------------------------------------ identity weights
__global__ void pack_identity_kernel(int channels, __nv_bfloat16* __restrict__ dst, long long nvec) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= nvec) return;
  const int r = (int)(id & 7), n8 = (int)((id >> 3) & 15), k8 = (int)((id >> 7) & 1);
  const long long rest = id >> 8;
  const int ksteps = channels / 16;
  const int ks = (int)(rest % ksteps), ntile = (int)(rest / ksteps);
  const int co = ntile * 128 + n8 * 8 + r;
  const int ci0 = ks * 16 + k8 * 8;
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) o[e] = pack_bf16x2(co == ci0 + 2 * e ? 1.f : 0.f, co == ci0 + 2 * e + 1 ? 1.f : 0.f);
  reinterpret_cast<uint4*>(dst)[id] = make_uint4(o[0], o[1], o[2], o[3]);
}
cudaError_t launch_pack_identity(int channels, __nv_bfloat16* dst, cudaStream_t s) {
  const long long nvec = (long long)(channels / 128) * (channels / 16) * 256;
  pack_identity_kernel<<<(unsigned)((nvec + 255) / 256), 256, 0, s>>>(channels, dst, nvec);
  return cudaGetLastError();
}

}  // namespace b200ad
