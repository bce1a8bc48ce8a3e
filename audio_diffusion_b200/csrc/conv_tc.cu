// wgmma implicit-GEMM convolution for the U-Net hot path (replaces the cuDNN conv2d calls that
// diffusers' UNet2DModel.forward makes; reference call site audiodiffusion/pipeline_audio_diffusion.py:163).
//
// GEMM view (transposed): D^T[cout, pixel] = sum over (segment, tap, cin) W[cout, cin, tap] * X[pixel + shift(tap), cin].
//   M = 128 output channels (weights are the A operand; two consumer warpgroups take 64 rows each), N = up to 256 output
//   pixels (activations are the B operand), K = 16 input channels per wgmma.m64nNk16.  The accumulators of an item
//   (64 x 256 fp32 per warpgroup) live in registers, which caps an item at two 128-pixel tiles.
// Pixel operand: the PF8 layout stores 8-channel vectors of consecutive pixels contiguously, which *is* the K-major
//   no-swizzle core-matrix layout (8 rows x 16 B). A work item covers 2 x 128 consecutive flat pixels; per 16 input
//   channels ONE contiguous window per 8-channel plane (the run plus a halo of Wp+1 pixels on both sides) is bulk-copied
//   (TMA engine) into shared memory, and every tap is a descriptor whose start address is shifted by (dh*Wp + dw) * 16 B.
//   (Few large copies: a bulk copy has a fixed cost however small it is.)
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
//   of a plane in lanes 4 apart, which is exactly a transposed 8x8 matrix) -> one bulk store (TMA engine) per plane and
//   tile, draining while the next item is multiplied.  Pad columns and the run-off behind the image are stored as the
//   zeros the layout requires there.
// Small images (H * Wp + bottom halo <= 128 pixels: 8x8 and below): an item's tiles are the first tiles of CONSECUTIVE
//   IMAGES, so one weight fetch and one N = 256 MMA serve two samples (ConvParams::pack).
// Warp roles (12 warps): 0 activation producer, 1 weight producer, 2-3 transform, 4-7 and 8-11 the two consumer
//   warpgroups (MMA + epilogue).
#include <cstdlib>

#include "conv_tc.cuh"

namespace b200ad {

constexpr int CONV_THREADS = 384;     // 12 warps
constexpr int CONV_XF_THREADS = 64;   // transform warps 2, 3
// epilogue staging, one buffer per consumer warpgroup: its 8 planes (64 channels) x 256 pixels, bf16
constexpr int CONV_SPLANE = CONV_MAXG * CONV_TM * 16;   // bytes per 8-channel plane of a buffer
constexpr int CONV_STG_WG = 8 * CONV_SPLANE;
constexpr int CONV_STAGING = 2 * CONV_STG_WG;

struct WorkItem {
  int n, ntile, m0, G;
};

__device__ __forceinline__ WorkItem decode_work(const ConvParams& p, int w) {
  WorkItem wi;
  wi.ntile = w % p.ntiles_n;
  const int gidx = w / p.ntiles_n;
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

__global__ void __launch_bounds__(CONV_THREADS, 1) conv_tc_kernel(const __grid_constant__ ConvParams p) {
  constexpr int ASM = CONV_AS_MAX, BSM = CONV_BS_MAX;
  const int AS = p.as;      // activation stages of this launch (CONV_AS .. CONV_AS_MAX)
  const int BS = p.bs;      // weight-ring depth of this launch (whatever the activation stages leave, CONV_BS .. CONV_BS_MAX)
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5;
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
  if (p.pdl) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (warp != 1) asm volatile("griddepcontrol.wait;" ::: "memory");
  }

  if (warp == 0) {
    // ================================ activation producer: per k-step two windows (one per 8-channel plane), lanes 0 / 1
    int stage = 0;
    uint32_t phase = 0;
    if (p.dbg & 4) {   // experiment: start the CTAs out of phase so that their epilogue store bursts do not coincide
      const long long t0 = clock64(), wait = (long long)(blockIdx.x & 7) * 2304;
      while (clock64() - t0 < wait) {}
    }
    for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
      const WorkItem wi = decode_work(p, w);
      for (int it = 0; it < p.ktotal; ++it) {
        const int ks = p.sched[it] & 255;
        const ConvSeg& sg = p.seg[p.sched[it] >> 8];
        const int npix = wi.G * CONV_TM + (sg.ht + sg.hb) * p.Wp + sg.hl + sg.hr;
        const uint32_t row_bytes = (uint32_t)npix * 16u;
        const uint32_t full = bar_fullA + 8 * stage;
        if (lane == 0) {
          mbar_wait(bar_emptyA + 8 * stage, phase ^ 1);
          mbar_arrive_expect_tx(full, 2u * row_bytes);
        }
        __syncwarp();
        const long long plane = (long long)(2 * ks + (lane & 1)) * p.PL;     // this lane's 8-channel plane of the k-step
        if (!p.pack) {
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
  } else if (warp == 1) {
    // ================================ weight producer: slots of up to CONV_BT taps (12 KB), one bulk copy each
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
        const int ntile = w % p.ntiles_n;
        for (int it = 0; it < p.ktotal; ++it) {
          const int ks = p.sched[it] & 255;
          const ConvSeg& sg = p.seg[p.sched[it] >> 8];
          const char* src = reinterpret_cast<const char*>(sg.wpack + (long long)ntile * sg.wtile_stride +
                                                          (long long)ks * sg.ntaps * (CONV_B_TAP / 2));
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
      for (int kidx = 0; kidx < p.ktotal; ++kidx) {
        const ConvSeg& sg = p.seg[p.sched[kidx] >> 8];
        const int npix = wi.G * CONV_TM + (sg.ht + sg.hb) * p.Wp + sg.hl + sg.hr;
        const uint32_t xlbo = (uint32_t)npix * 16u;   // the second 8-channel plane of the window
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
            const uint64_t xdesc = gmma_desc(abase + (uint32_t)sg.aoff[t0 + t] * 16u, xlbo, 128);
            if (wi.G == 2) wgmma_m64n256k16<0, 0>(acc, wdesc, xdesc);
            else           wgmma_m64n128k16<0, 0>(acc, wdesc, xdesc);
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous group has retired: its slots are free
          release();
          pend_b = sb;
          pend_a = (t0 + CONV_BT >= ntaps) ? sa : -1;
          if (++sb == BS) { sb = 0; pb ^= 1; }
        }
        if (++sa == AS) { sa = 0; pa ^= 1; }
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
                // and do not count for the statistics
                const int col1 = (col + 1 == p.Wp) ? 0 : col + 1;
                const bool v0 = m < hw_end && col < p.W, v1 = m + 1 < hw_end && col1 < p.W;
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
      if (!p.up2) {
        fence_proxy_async_smem();   // staging rows written through the generic proxy -> visible to the TMA engine
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
        // folded upsample: scatter into the 2x tensor at this launch's parity, straight from the staging rows
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
    const int xg0 = warp - 2;
    constexpr int xng = 1;
    constexpr int XSWEEP = CONV_XF_THREADS;
    int stage = 0;
    uint32_t phase = 0;
    for (int w = blockIdx.x; w < p.total_work; w += gridDim.x) {
      const WorkItem wi = decode_work(p, w);
      int last_s = -1, npix = 0, drow = 0, dcol = 0;
      const float2* ssn = nullptr;
      bool silu = false;
      int row0[2] = {0, 0}, col0[2] = {0, 0};
      for (int it = 0; it < p.ktotal; ++it) {
        const int ks = p.sched[it] & 255, s = p.sched[it] >> 8;
        const ConvSeg& sg = p.seg[s];
        if (s != last_s) {     // per-segment state (the schedule may alternate between segments)
          last_s = s;
          npix = wi.G * CONV_TM + (sg.ht + sg.hb) * p.Wp + sg.hl + sg.hr;
          ssn = sg.ss ? sg.ss + (long long)wi.n * sg.ss_stride : nullptr;
          // flat position of this thread's first pixel(s); (row, col) advance incrementally (one sweep per iteration)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int m_first = wi.m0 - sg.ht * p.Wp - sg.hl + (xg0 + u) * 32 + lane;
            row0[u] = (m_first >= 0) ? m_first / p.Wp : -1 - ((-1 - m_first) / p.Wp);  // floor division
            col0[u] = m_first - row0[u] * p.Wp;
          }
          drow = XSWEEP / p.Wp;
          dcol = XSWEEP - drow * p.Wp;
          silu = sg.silu != 0;
        }
        {
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
            const int tidx = (warp - 2) * 32 + lane;
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
            int row[2] = {row0[0], row0[1]}, col[2] = {col0[0], col0[1]};
            for (int px0 = xg0 * 32 + lane; px0 < npix; px0 += XSWEEP) {
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                if (u < xng) {
                  const int px = px0 + u * 32;
                  if (px < npix) {
                    const bool valid = (row[u] >= 0) && (row[u] < p.H) && (col[u] < p.W);
                    uint4 a = make_uint4(0, 0, 0, 0), b = make_uint4(0, 0, 0, 0);
                    if (valid) {
                      a = base[px];
                      b = base[npix + px];
                      if (silu) { a = xform_vec<true>(a, sc0, sh0); b = xform_vec<true>(b, sc1, sh1); }
                      else      { a = xform_vec<false>(a, sc0, sh0); b = xform_vec<false>(b, sc1, sh1); }
                    }
                    base[px] = a;
                    base[npix + px] = b;
                  }
                  row[u] += drow; col[u] += dcol;
                  if (col[u] >= p.Wp) { col[u] -= p.Wp; ++row[u]; }
                }
              }
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

cudaError_t launch_conv_tc(const ConvParams& p_in, int num_sms, cudaStream_t stream) {
  // timing experiments only; read on every launch so that one process can alternate settings (tools/ab_conv.py)
  const char* dbg_env = getenv("B200AD_CONV_DBG");
  const int dbg = dbg_env ? atoi(dbg_env) : 0;
  if (p_in.nseg < 1 || p_in.nseg > CONV_MAXSEG) return cudaErrorInvalidValue;
  ConvParams p = p_in;
  p.dbg = dbg;
  for (int s = 0; s < p.nseg; ++s)
    if (p.seg[s].wtile_stride == 0) p.seg[s].wtile_stride = (long long)p.seg[s].ksteps * p.seg[s].ntaps * (CONV_B_TAP / 2);
  // Experiment (B200AD_CONV_DBG & 128, off by default): move trailing 1-tap segments (shortcut / residual) in front of the
  // main segment's last k-step so that a many-tap k-step closes the K loop.  The 1-tap k-steps are load-bound (a 16 KB
  // window per k-step of MMAs) and would stall the ring in the middle of the item instead of next to the epilogue.
  if ((dbg & 128) && p.nseg >= 2 && p.nseg < CONV_MAXSEG && p.seg[0].ksteps >= 2 && p.seg[p.nseg - 1].ntaps < p.seg[0].ntaps) {
    ConvSeg tail = p.seg[0];
    const int ka = tail.ksteps - 1;
    p.seg[0].ksteps = ka;
    tail.ksteps = 1;
    tail.src += (long long)ka * 2 * p.PL * 8;
    tail.wpack += (long long)ka * tail.ntaps * (CONV_B_TAP / 2);
    if (tail.ss) tail.ss += ka * 16;
    p.seg[p.nseg++] = tail;
  }
  p.ktotal = 0;
  for (int s = 0; s < p.nseg; ++s) {
    if (p.seg[s].ksteps > 255) return cudaErrorInvalidValue;
    p.ktotal += p.seg[s].ksteps;
  }
  if (p.ktotal > CONV_MAXSCHED) return cudaErrorInvalidValue;
  {
    // heavy = many-tap k-steps in segment order, light = 1-tap k-steps in segment order; light ones are spread evenly over
    // the gaps between heavy ones
    int nh = 0, nl = 0;
    for (int s = 0; s < p.nseg; ++s) (p.seg[s].ntaps > 1 ? nh : nl) += p.seg[s].ksteps;
    int n = 0;
    // (interleaving is an experiment switch, B200AD_CONV_DBG & 2048, not the default)
    if (!(dbg & 2048) || nh < 2 || nl == 0) {
      for (int s = 0; s < p.nseg; ++s)
        for (int ks = 0; ks < p.seg[s].ksteps; ++ks) p.sched[n++] = (unsigned short)((s << 8) | ks);
    } else {
      int hs = 0, hk = 0, ls = 0, lk = 0;      // cursors (segment, k-step) into the heavy / light sequences
      auto next = [&](bool heavy, int& cs, int& ck) {
        while ((p.seg[cs].ntaps > 1) != heavy || ck >= p.seg[cs].ksteps) { ++cs; ck = 0; }
        p.sched[n++] = (unsigned short)((cs << 8) | ck);
        ++ck;
      };
      int emitted_light = 0;
      for (int i = 0; i < nh; ++i) {
        next(true, hs, hk);
        if (i < nh - 1) {
          const int want = (int)((long long)(i + 1) * nl / (nh - 1));     // light k-steps due after heavy k-step i
          for (; emitted_light < want; ++emitted_light) next(false, ls, lk);
        }
      }
    }
  }
  p.groups_per_img = (p.H * p.Wp + CONV_MAXG * CONV_TM - 1) / (CONV_MAXG * CONV_TM);
  p.ntiles_n = p.cout / CONV_NT;
  p.total_work = p.N * p.groups_per_img * p.ntiles_n;
  // Small images (8x8 and below at the bottom of the U-Net, every level of the latent model below 16x16): one image is a
  // fraction of a tile, so an item per image fetches the full weight set (1.2 MB for 512 -> 512) for <= 72 pixels and runs
  // N = 128 MMAs.  Packed, an item holds the first tile of up to four consecutive images: the window of tile g is image
  // n + g's plane from its pixel 0 on, whose tail is that image's own zero guard, so every tap of a valid output pixel stays
  // inside its tile (needs H * Wp + the bottom halo <= 128) and the MMA issue is unchanged.
  p.pack = 0;
  if (!(dbg & 256)) {
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
  }
  // the two windows of one k-step must fit an activation slot
  int a_stage = 0;
  const int tiles_img = (p.H * p.Wp + CONV_TM - 1) / CONV_TM;
  const int max_g = p.pack ? p.pack : (tiles_img < CONV_MAXG ? tiles_img : CONV_MAXG);   // most tiles any item of this launch has
  for (int s = 0; s < p.nseg; ++s) {
    const ConvSeg& sg = p.seg[s];
    const int npix = max_g * CONV_TM + (sg.ht + sg.hb) * p.Wp + sg.hl + sg.hr;
    a_stage = npix * 32 > a_stage ? npix * 32 : a_stage;
    if (sg.ntaps > CONV_MAXTAPS || sg.ntaps > CONV_BT * (CONV_BS - 1) || npix > 0x3FFF) return cudaErrorInvalidValue;
    for (int t = 0; t < sg.ntaps; ++t) p.seg[s].aoff[t] = (sg.dh[t] + sg.ht) * p.Wp + sg.dw[t] + sg.hl;
  }
  p.a_stage = (a_stage + 255) & ~255;
  // Ring depths: W = 256 fills shared memory with 3 activation stages + 5 weight slots.  Launches with smaller windows (narrow
  // images, packed small images, 1-tap convs) have SHORT k-steps, and the TMA -> transform -> MMA chain of a stage (a few
  // thousand cycles of L2 latency) is then covered only by more stages in flight: first up to 6 activation stages, then the
  // weight ring up to its maximum, then the remaining activation stages.
  p.as = CONV_AS;
  p.bs = CONV_BS;
  if (!(dbg & 512)) {
    auto fits = [&](int as, int bs) {
      // 1 KB of head room: the kernel's static shared memory counts against the same 227 KB
      return (size_t)as * p.a_stage + (size_t)bs * CONV_B_SLOT + CONV_STAGING + 2048 <= (size_t)CONV_SMEM_MAX;
    };
    while (p.as < 6 && fits(p.as + 1, p.bs)) ++p.as;
    while (p.bs < CONV_BS_MAX && fits(p.as, p.bs + 1)) ++p.bs;
    while (p.as < CONV_AS_MAX && fits(p.as + 1, p.bs)) ++p.as;
  }
  const size_t smem = (size_t)p.as * p.a_stage + (size_t)p.bs * CONV_B_SLOT + CONV_STAGING + 1024;
  if (smem > (size_t)CONV_SMEM_MAX) return cudaErrorInvalidValue;  // image too wide for this tiling
  const int grid = p.total_work < num_sms ? p.total_work : num_sms;
  if (grid <= 0) return cudaSuccess;
  static size_t attr = 0;
  if (smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = smem;
  }
  p.pdl = (dbg & 1024) ? 0 : 1;
  if (!p.pdl) {
    conv_tc_kernel<<<grid, CONV_THREADS, smem, stream>>>(p);
    return cudaGetLastError();
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
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel, p);
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
