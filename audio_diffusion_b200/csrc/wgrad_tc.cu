// Weight gradient of a convolution on wgmma.
//   dW[co][ci][tap] = sum over samples and flat pixels p of  gY[co][p] * A[ci][p + shift(tap)]
// GEMM view per tap: D[M = 128 co][N = NCI ci] += sum_K gY[co][K = pixel] * A[ci][K = pixel + shift]: the reduction runs over
// PIXELS, so both operands are "MN-major": in PF8 the 8 channels of a pixel are contiguous (MN) and consecutive pixels are
// 16 B apart (K) — a run of 8 pixels of one 8-channel plane IS the 8x8 MN-major core matrix (128 B): LBO (next 8 pixels) =
// 128 B, SBO (next 8 channels) = the plane pitch of the staged window.
// Work decomposition: one CTA = (128-co tile, NCI-ci tile, ONE ROW of taps (same dh, dw in {-1,0,+1}), a share of the pixel
// blocks).  A tap row needs only a 1-pixel halo (the row offset dh*Wp moves the window start), and its <= 3 taps are shifted
// descriptors of one activation window.  Two consumer warpgroups take 64 output channels each and keep 3 taps x NCI fp32
// accumulators in registers across all of the CTA's pixel blocks.  Partial dW is added to global memory with fp32 atomics
// (split-K over pixels and CTAs).
#include <cstdlib>

#include "bwd_kernels.cuh"
#include "conv_tc.cuh"

namespace b200ad {

struct WgradParams {
  const __nv_bfloat16* gy;    // PF8 view, cout channels
  const __nv_bfloat16* act;   // PF8 view, cin channels (the conv's input as the forward pass saw it)
  float* dw;                  // fp32, element (co, ci, t) at (co * cin_total + ci_off + ci) * ntaps_total + tapidx
  int N, H, W, Wp, lead, PL, cin, cout;
  int gy_img_planes, act_img_planes, cin_total, ci_off, ntaps_total;
  int nrows;                  // tap rows (distinct dh)
  int row_off[3];             // dh * Wp of the row
  int row_ntaps[3];
  int row_dw[3][3];           // dw of each tap of the row
  int row_tapidx[3][3];       // destination tap index
  int P;                      // pixels per staged block (multiple of 16)
  int nblk;                   // blocks per image
};

constexpr int WG_THREADS = 288;   // warps 0-3 and 4-7: consumer warpgroups (MMA + epilogue), warp 8: producer

template <int NCI, int STAGES>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tc_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gy_bytes = p.P * 256;                             // 16 planes x P pixels x 16 B
  const int act_pix = p.P + 2;                                // 1-pixel halo on both sides
  const int act_bytes = (NCI / 8) * act_pix * 16;
  const int stage_bytes = (gy_bytes + act_bytes + 127) & ~127;
  uint8_t* ctrl = smem + STAGES * stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ctrl);         // full[S], empty[S]
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + STAGES);
  if (warp == 8 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 8); }
    mbar_fence_init();
  }
  __syncthreads();
  const int row = blockIdx.y % p.nrows, cj = blockIdx.y / p.nrows, ct = blockIdx.z;
  const int total_blocks = p.N * p.nblk;
  const int ntaps = p.row_ntaps[row];

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int roff = p.row_off[row];
      for (int b = blockIdx.x; b < total_blocks; b += gridDim.x) {
        const int n = b / p.nblk, m0 = (b - n * p.nblk) * p.P;
        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
        mbar_arrive_expect_tx(bar_full + 8 * stage, (uint32_t)(gy_bytes + act_bytes));
        const uint32_t dst = smem_base + stage * stage_bytes;
        for (int pl = 0; pl < 16; ++pl) {
          const __nv_bfloat16* src = p.gy + (((long long)n * p.gy_img_planes + ct * 16 + pl) * p.PL + p.lead + m0) * 8;
          bulk_g2s(dst + pl * p.P * 16, src, (uint32_t)p.P * 16u, bar_full + 8 * stage);
        }
        for (int pl = 0; pl < NCI / 8; ++pl) {
          const __nv_bfloat16* src =
              p.act + (((long long)n * p.act_img_planes + cj * (NCI / 8) + pl) * p.PL + p.lead + m0 + roff - 1) * 8;
          bulk_g2s(dst + gy_bytes + pl * act_pix * 16, src, (uint32_t)act_pix * 16u, bar_full + 8 * stage);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // consumer warpgroup cw: output channels [64 cw, 64 cw + 64) of the co tile.  Accumulator fragment of tap t: warp wq,
    // lane l holds co 16 wq + l/4 (+8) and ci 8j + 2 (l % 4) (+1) in acc[t][4j + {0, 1}] (co + 8: acc[t][4j + {2, 3}]).
    const int cw = warp >> 2, wq = warp & 3;
    float acc[3][NCI / 2];
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int i = 0; i < NCI / 2; ++i) acc[t][i] = 0.f;
    const uint32_t a_sbo = (uint32_t)p.P * 16u, b_sbo = (uint32_t)act_pix * 16u;
    const uint32_t dw0 = (uint32_t)(p.row_dw[row][0] + 1) * 16u, dw1 = (uint32_t)(p.row_dw[row][1] + 1) * 16u,
                   dw2 = (uint32_t)(p.row_dw[row][2] + 1) * 16u;   // + halo
    int stage = 0;
    uint32_t phase = 0;
    for (int b = blockIdx.x; b < total_blocks; b += gridDim.x) {
      mbar_wait(bar_full + 8 * stage, phase);
      const uint32_t a0 = smem_base + stage * stage_bytes + (uint32_t)cw * 8u * a_sbo;   // planes 8 cw .. 8 cw + 7 of gY
      const uint32_t b0 = smem_base + stage * stage_bytes + (uint32_t)gy_bytes;
      const int ksteps = p.P / 16;
      wgmma_fence();
      for (int k = 0; k < ksteps; ++k) {
        const uint64_t adesc = gmma_desc(a0 + (uint32_t)k * 256u, 128, a_sbo);
        const uint32_t bk = b0 + (uint32_t)k * 256u;
        if (NCI == 64) wgmma_m64n64k16<1, 1>(acc[0], adesc, gmma_desc(bk + dw0, 128, b_sbo));
        else           wgmma_m64n32k16<1, 1>(acc[0], adesc, gmma_desc(bk + dw0, 128, b_sbo));
        if (ntaps > 1) {
          if (NCI == 64) wgmma_m64n64k16<1, 1>(acc[1], adesc, gmma_desc(bk + dw1, 128, b_sbo));
          else           wgmma_m64n32k16<1, 1>(acc[1], adesc, gmma_desc(bk + dw1, 128, b_sbo));
        }
        if (ntaps > 2) {
          if (NCI == 64) wgmma_m64n64k16<1, 1>(acc[2], adesc, gmma_desc(bk + dw2, 128, b_sbo));
          else           wgmma_m64n32k16<1, 1>(acc[2], adesc, gmma_desc(bk + dw2, 128, b_sbo));
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * stage);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if (blockIdx.x < total_blocks) {
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        if (t < ntaps) {
          const int tapidx = p.row_tapidx[row][t];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int co = ct * 128 + cw * 64 + wq * 16 + 8 * h + (lane >> 2);
            float* dst = p.dw + ((long long)co * p.cin_total + p.ci_off + cj * NCI + 2 * (lane & 3)) * p.ntaps_total + tapidx;
#pragma unroll
            for (int j = 0; j < NCI / 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                atomicAdd(dst + (long long)(8 * j + e) * p.ntaps_total, acc[t][4 * j + 2 * h + e]);
          }
        }
      }
    }
  }
}

template <int NCI, int STAGES>
static cudaError_t launch_wg(const WgradParams& p, int num_sms, cudaStream_t s) {
  const int act_pix = p.P + 2;
  const int stage_bytes = (p.P * 256 + (NCI / 8) * act_pix * 16 + 127) & ~127;
  const size_t smem = (size_t)STAGES * stage_bytes + 256;
  if (smem > (size_t)CONV_SMEM_MAX) return cudaErrorInvalidValue;
  auto kern = wgrad_tc_kernel<NCI, STAGES>;
  static size_t attr = 0;
  if (smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr = smem;
  }
  const int tiles = p.nrows * (p.cin / NCI) * (p.cout / 128);
  int splits = num_sms / tiles;
  if (splits < 1) splits = 1;
  if (splits > p.N * p.nblk) splits = p.N * p.nblk;
  dim3 grid(splits, p.nrows * (p.cin / NCI), p.cout / 128);
  kern<<<grid, WG_THREADS, smem, s>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_wgrad_tc(const WgradDesc& d, int num_sms, cudaStream_t s) {
  if (d.cout % 128 || d.cin % 32 || d.ntaps < 1 || d.ntaps > 9) return cudaErrorInvalidValue;
  const Geom g = make_geom(d.N, d.H, d.W);
  WgradParams p{};
  p.gy = d.gy; p.act = d.act; p.dw = d.dw;
  p.N = d.N; p.H = d.H; p.W = d.W; p.Wp = g.Wp; p.lead = g.lead; p.PL = g.PL; p.cin = d.cin; p.cout = d.cout;
  p.gy_img_planes = d.gy_img_planes; p.act_img_planes = d.act_img_planes;
  p.cin_total = d.cin_total; p.ci_off = d.ci_off; p.ntaps_total = d.ntaps_total;
  // group the taps into rows of equal dh
  p.nrows = 0;
  for (int t = 0; t < d.ntaps; ++t) {
    if (d.dh[t] < -1 || d.dh[t] > 1 || d.dw_[t] < -1 || d.dw_[t] > 1) return cudaErrorInvalidValue;
    int r = -1;
    for (int k = 0; k < p.nrows; ++k)
      if (p.row_off[k] == d.dh[t] * g.Wp) r = k;
    if (r < 0) {
      if (p.nrows == 3) return cudaErrorInvalidValue;
      r = p.nrows++;
      p.row_off[r] = d.dh[t] * g.Wp;
      p.row_ntaps[r] = 0;
    }
    if (p.row_ntaps[r] == 3) return cudaErrorInvalidValue;
    p.row_dw[r][p.row_ntaps[r]] = d.dw_[t];
    p.row_tapidx[r][p.row_ntaps[r]] = d.tapidx[t];
    ++p.row_ntaps[r];
  }
  const int flat = d.H * g.Wp;
  if (d.cin % 64 == 0) {
    // 64-wide ci tiles (3 taps x 32 accumulator registers per ci tile and thread): 192-pixel stages, two of them (2 x 73 KB)
    p.P = flat <= 128 ? 128 : 192;
    p.nblk = (flat + p.P - 1) / p.P;
    return launch_wg<64, 2>(p, num_sms, s);
  }
  p.P = flat <= 128 ? 128 : 256;
  p.nblk = (flat + p.P - 1) / p.P;
  return launch_wg<32, 2>(p, num_sms, s);
}

}  // namespace b200ad
