// SIMT kernels of the U-Net path that are HBM-bound or degenerate for tensor cores:
// weight packing, GroupNorm(+SiLU) apply, conv_in (Cin = 1), conv_norm_out + conv_out (Cout = 1) fused with
// the DDPM/DDIM update, nearest-2x upsample, stride-2 parity split and layout conversion.
// Reference semantics: diffusers UNet2DModel / DDPMScheduler.step / DDIMScheduler.step as called from
// audiodiffusion/pipeline_audio_diffusion.py:163-179 (restated in oracle/unet_oracle.py, oracle/schedulers_oracle.py).
#include <cstring>

#include "kernels.cuh"

namespace b200ad {

// ------------------------------------------------------------------------------------ weight packing
__device__ __forceinline__ void pack_one_vector(const float* __restrict__ w, int cout, int cin_total, int KH, int KW,
                                                int cin_off, int ksteps, const PackTaps& taps,
                                                __nv_bfloat16* __restrict__ dst, long long id, int cout_real) {
  const int r = (int)(id & 7);
  const int n8 = (int)((id >> 3) & 15);
  const int k8 = (int)((id >> 7) & 1);
  long long rest = id >> 8;
  const int tap = (int)(rest % taps.ntaps);
  rest /= taps.ntaps;
  const int ks = (int)(rest % ksteps);
  const int ntile = (int)(rest / ksteps);
  const int co = ntile * 128 + n8 * 8 + r;
  const int ci0 = cin_off + ks * 16 + k8 * 8;
  float v[8];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const float* wp = taps.transpose ? w + ((long long)(ci0 + kk) * cout_real + co) * KH * KW
                                     : w + ((long long)co * cin_total + ci0 + kk) * KH * KW;
    float a = 0.f;
    if (co >= cout_real) {
      // rows beyond the real output channels (cout padded to the 128-channel tile) are zero
    } else if (taps.fold) {
      const unsigned mask = taps.fold_mask[tap];
      for (int t = 0; t < KH * KW; ++t)
        if (mask & (1u << t)) a += wp[t];
    } else {
      a = wp[taps.kh[tap] * KW + taps.kw[tap]];
    }
    v[kk] = a;
  }
  uint4 o;
  o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
  o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
  reinterpret_cast<uint4*>(dst)[id] = o;
}

__global__ void pack_weights_kernel(const float* __restrict__ w, int cout, int cin_total, int KH, int KW, int cin_off,
                                    int ksteps, PackTaps taps, __nv_bfloat16* __restrict__ dst, long long nvec, int cout_real) {
  const long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= nvec) return;
  pack_one_vector(w, cout, cin_total, KH, KW, cin_off, ksteps, taps, dst, id, cout_real);
}

// one launch for a whole job table: block b packs vectors [256 * first, 256 * first + 256) of job blk[b].x
__global__ void __launch_bounds__(256) pack_batch_kernel(const PackItem* __restrict__ items, const int2* __restrict__ blk) {
  __shared__ PackItem it;
  const int2 bj = blk[blockIdx.x];
  if (threadIdx.x == 0) it = items[bj.x];
  __syncthreads();
  const long long id = (long long)bj.y * 256 + threadIdx.x;
  if (id >= it.nvec) return;
  pack_one_vector(it.w, it.cout, it.cin_total, it.KH, it.KW, it.cin_off, it.ksteps, it.taps, it.dst, id, it.cout_real);
}

PackBatch::~PackBatch() {
  if (d_items) cudaFree(d_items);
  if (d_blk) cudaFree(d_blk);
}

cudaError_t launch_pack_batch(PackBatch& pb, const std::vector<PackItem>& items, cudaStream_t s) {
  if (items.empty()) return cudaSuccess;
  const bool same = pb.host.size() == items.size() &&
                    memcmp(pb.host.data(), items.data(), items.size() * sizeof(PackItem)) == 0;
  if (!same) {
    std::vector<int2> blk;
    for (size_t j = 0; j < items.size(); ++j) {
      const int nb = (int)((items[j].nvec + 255) / 256);
      for (int b = 0; b < nb; ++b) blk.push_back(make_int2((int)j, b));
    }
    cudaError_t e = cudaStreamSynchronize(s);          // the old tables may still be in use
    if (e != cudaSuccess) return e;
    if (pb.d_items) cudaFree(pb.d_items);
    if (pb.d_blk) cudaFree(pb.d_blk);
    pb.d_items = pb.d_blk = nullptr;
    if ((e = cudaMalloc(&pb.d_items, items.size() * sizeof(PackItem))) != cudaSuccess) return e;
    if ((e = cudaMalloc(&pb.d_blk, blk.size() * sizeof(int2))) != cudaSuccess) return e;
    if ((e = cudaMemcpy(pb.d_items, items.data(), items.size() * sizeof(PackItem), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    if ((e = cudaMemcpy(pb.d_blk, blk.data(), blk.size() * sizeof(int2), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    pb.host = items;
    pb.nblocks = (int)blk.size();
  }
  pack_batch_kernel<<<pb.nblocks, 256, 0, s>>>((const PackItem*)pb.d_items, (const int2*)pb.d_blk);
  return cudaGetLastError();
}

cudaError_t launch_pack_weights(const float* w, int cout, int cin_total, int KH, int KW, int cin_off, int ksteps,
                                const PackTaps& taps, __nv_bfloat16* dst, cudaStream_t s, int cout_real) {
  const long long nvec = (long long)(cout / 128) * ksteps * taps.ntaps * 256;
  const int threads = 256;
  const long long blocks = (nvec + threads - 1) / threads;
  pack_weights_kernel<<<(unsigned)blocks, threads, 0, s>>>(w, cout, cin_total, KH, KW, cin_off, ksteps, taps, dst, nvec,
                                                             cout_real < 0 ? cout : cout_real);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ GroupNorm apply
// Materialised GroupNorm(+SiLU) (the weight-gradient kernel's activation operand in the backward pass; the forward pass
// applies the norm inside conv_tc_kernel).  grid (position chunks, planes, N): a CTA walks a flat run of one 8-channel plane
// (coalesced 16-byte vectors, 4 in flight per thread); eight threads derive the plane's scale / shift from the fp64 sums.
constexpr int GN_CHUNK = 8192;

__global__ void __launch_bounds__(256) gn_apply_kernel(const GnApplyParams p) {
  __shared__ float coef[2][8];
  const int Ct = p.C[0] + p.C[1];
  const int n = blockIdx.z, pl = blockIdx.y;
  const int cpg = Ct / p.groups;
  const Geom g = make_geom(p.N, p.H, p.W);
  if (threadIdx.x < 8) {
    const int c = pl * 8 + threadIdx.x, gi = c / cpg;
    double s = 0., q = 0.;
    for (int cc = gi * cpg; cc < (gi + 1) * cpg; cc += 4) {
      const stat_t* st = (cc < p.C[0]) ? p.stats[0] + ((long long)n * (p.C[0] >> 2) + (cc >> 2)) * 2
                                      : p.stats[1] + ((long long)n * (p.C[1] >> 2) + ((cc - p.C[0]) >> 2)) * 2;
      s += st[0];
      q += st[1];
    }
    const double cnt = (double)cpg * (double)p.H * (double)p.W;
    const double mean = s / cnt;
    const float rstd = (float)(1.0 / sqrt(fmax(q / cnt - mean * mean, 0.) + (double)p.eps));
    const float sc = p.gamma[c] * rstd;
    const float hs = p.silu ? 0.5f : 1.0f;    // SiLU works on a / 2: silu(a) = h + h tanh(h), h = a / 2
    coef[0][threadIdx.x] = sc * hs;
    coef[1][threadIdx.x] = (p.beta[c] - (float)mean * sc) * hs;
  }
  __syncthreads();
  float sc[8], sh[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { sc[e] = coef[0][e]; sh[e] = coef[1][e]; }
  const int planes0 = p.C[0] >> 3;
  const __nv_bfloat16* sp = (pl < planes0) ? p.src[0] + ((long long)n * planes0 + pl) * g.PL * 8
                                          : p.src[1] + ((long long)n * (p.C[1] >> 3) + (pl - planes0)) * g.PL * 8;
  const uint4* xv4 = reinterpret_cast<const uint4*>(sp) + g.lead;
  uint4* dv4 = reinterpret_cast<uint4*>(p.dst + ((long long)n * (Ct >> 3) + pl) * g.PL * 8) + g.lead;
  const int mend = min(p.H * g.Wp, (int)(blockIdx.x + 1) * GN_CHUNK);
  int m0 = blockIdx.x * GN_CHUNK + threadIdx.x;
  int col = m0 % g.Wp;
  const int dcol = 256 % g.Wp;
  for (; m0 < mend; m0 += 4 * 256) {
    uint4 xr[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * 256;
      xr[u] = (m < mend) ? xv4[m] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int m = m0 + u * 256;
      const bool pad = col == p.W;     // the pad column closing every row stays zero
      col += dcol;
      if (col >= g.Wp) col -= g.Wp;
      if (m >= mend) continue;
      const uint32_t w[4] = {xr[u].x, xr[u].y, xr[u].z, xr[u].w};
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(w[e]);
        float a = fmaf(f.x, sc[2 * e], sh[2 * e]);
        float b = fmaf(f.y, sc[2 * e + 1], sh[2 * e + 1]);
        if (p.silu) { a = fmaf(a, tanh_approx(a), a); b = fmaf(b, tanh_approx(b), b); }
        o[e] = pack_bf16x2(a, b);
      }
      dv4[m] = pad ? make_uint4(0, 0, 0, 0) : make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

cudaError_t launch_gn_apply(const GnApplyParams& p, cudaStream_t s) {
  const int Ct = p.C[0] + p.C[1];
  if (Ct % p.groups) return cudaErrorInvalidValue;
  const dim3 grid((p.H * (p.W + 1) + GN_CHUNK - 1) / GN_CHUNK, Ct >> 3, p.N);
  gn_apply_kernel<<<grid, 256, 0, s>>>(p);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ GroupNorm finalize
// quad sums (one or two concatenated sources) -> per-(sample, channel) scale = gamma * rstd, shift = beta - mean * scale,
// consumed by the transform warps of conv_tc_kernel.  grid (N), 256 threads.
__global__ void __launch_bounds__(256) gn_finalize_kernel(const GnApplyParams p, float2* __restrict__ ss) {
  __shared__ float gmean[64], grstd[64];
  const int Ct = p.C[0] + p.C[1];
  const int n = blockIdx.x;
  const int cpg = Ct / p.groups;
  for (int gi = threadIdx.x; gi < p.groups; gi += blockDim.x) {
    double s = 0., q = 0.;
    for (int c = gi * cpg; c < (gi + 1) * cpg; c += 4) {
      const stat_t* st = (c < p.C[0]) ? p.stats[0] + ((long long)n * (p.C[0] >> 2) + (c >> 2)) * 2
                                     : p.stats[1] + ((long long)n * (p.C[1] >> 2) + ((c - p.C[0]) >> 2)) * 2;
      s += st[0];
      q += st[1];
    }
    const double cnt = (double)cpg * (double)p.H * (double)p.W;
    const double mean = s / cnt;
    const double var = fmax(q / cnt - mean * mean, 0.);
    gmean[gi] = (float)mean;
    grstd[gi] = (float)(1.0 / sqrt(var + (double)p.eps));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Ct; c += blockDim.x) {
    const int gi = c / cpg;
    const float sc = p.gamma[c] * grstd[gi];
    ss[(long long)n * Ct + c] = make_float2(sc, p.beta[c] - gmean[gi] * sc);
  }
}
cudaError_t launch_gn_finalize(const GnApplyParams& p, float2* ss, cudaStream_t s) {
  if (p.groups > 64) return cudaErrorInvalidValue;
  gn_finalize_kernel<<<p.N, 256, 0, s>>>(p, ss);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ conv_in
// fp32 NCHW (cin small) -> raw bf16 PF8 + quad statistics. One CTA = one 8-channel plane x 1024 pixels; the 8 x cin x 9
// weights of the plane sit in registers, each thread produces CI_PIX pixels (HBM-write bound).
constexpr int CI_PIX = 2;
__global__ void __launch_bounds__(256) conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ b, int N, int cin, int H, int W,
                                                      int cout, __nv_bfloat16* __restrict__ out,
                                                      stat_t* __restrict__ stats) {
  __shared__ float red[8][4];
  const Geom g = make_geom(N, H, W);
  const int n = blockIdx.z, pl = blockIdx.y;
  float acc[CI_PIX][8];
  int hh0[CI_PIX], ww0[CI_PIX];
  bool ok[CI_PIX];
#pragma unroll
  for (int u = 0; u < CI_PIX; ++u) {
    const int pidx = (blockIdx.x * CI_PIX + u) * blockDim.x + threadIdx.x;
    ok[u] = pidx < H * W;
    hh0[u] = ok[u] ? pidx / W : 0;
    ww0[u] = ok[u] ? pidx - hh0[u] * W : 0;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[u][e] = __ldg(b + pl * 8 + e);
  }
  for (int ci = 0; ci < cin; ++ci) {
    float wr[8][9];
#pragma unroll
    for (int e = 0; e < 8; ++e)
#pragma unroll
      for (int t = 0; t < 9; ++t) wr[e][t] = __ldg(w + ((long long)(pl * 8 + e) * cin + ci) * 9 + t);
    const float* xi = x + ((long long)n * cin + ci) * H * W;
#pragma unroll
    for (int u = 0; u < CI_PIX; ++u) {
      float xv[9];
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int hh = hh0[u] + t / 3 - 1, wx = ww0[u] + t % 3 - 1;
        xv[t] = (ok[u] && hh >= 0 && hh < H && wx >= 0 && wx < W) ? __ldg(xi + hh * W + wx) : 0.f;
      }
#pragma unroll
      for (int t = 0; t < 9; ++t)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[u][e] = fmaf(xv[t], wr[e][t], acc[u][e]);
    }
  }
  float s4[4] = {0.f, 0.f, 0.f, 0.f};
  __nv_bfloat16* plane = out + ((long long)n * (cout >> 3) + pl) * g.PL * 8;
#pragma unroll
  for (int u = 0; u < CI_PIX; ++u) {
    if (!ok[u]) continue;
    const float* a = acc[u];
    uint4 o;
    o.x = pack_bf16x2(a[0], a[1]); o.y = pack_bf16x2(a[2], a[3]);
    o.z = pack_bf16x2(a[4], a[5]); o.w = pack_bf16x2(a[6], a[7]);
    *reinterpret_cast<uint4*>(plane + (long long)(g.lead + hh0[u] * g.Wp + ww0[u]) * 8) = o;
    s4[0] += a[0] + a[1] + a[2] + a[3];
    s4[1] += a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3];
    s4[2] += a[4] + a[5] + a[6] + a[7];
    s4[3] += a[4] * a[4] + a[5] * a[5] + a[6] * a[6] + a[7] * a[7];
  }
  if (stats) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int sh = 16; sh >= 1; sh >>= 1) s4[k] += __shfl_xor_sync(0xffffffffu, s4[k], sh);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[warp][0] = s4[0]; red[warp][1] = s4[1]; red[warp][2] = s4[2]; red[warp][3] = s4[3]; }
    __syncthreads();
    if (threadIdx.x < 4) {
      float t = 0.f;
      for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
      // quads 2*pl (values 0,1) and 2*pl+1 (values 2,3)
      stat_t* dst = stats + ((long long)n * (cout >> 2) + pl * 2 + (threadIdx.x >> 1)) * 2 + (threadIdx.x & 1);
      atomicAdd(dst, (stat_t)t);
    }
  }
}

// cin == 1, W % 4 == 0 (every U-Net / VAE-encoder input): the plane's 72 weights stay in registers while the CTA walks
// CIQ_ITER x 256 groups of 4 horizontally adjacent pixels; each group reads its 3 x 6 input patch once (vector load for the
// aligned middle) and the statistics are reduced once per CTA.  Same FMA order as conv_in_kernel (bit-identical outputs).
constexpr int CIQ_ITER = 4;
__global__ void __launch_bounds__(256, 2) conv_in_c1_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ b, int N, int H, int W, int cout,
                                                         __nv_bfloat16* __restrict__ out, stat_t* __restrict__ stats) {
  __shared__ float red[8][4];
  const Geom g = make_geom(N, H, W);
  const int n = blockIdx.z, pl = blockIdx.y;
  float bias[8];
  f32x2_t w2[4][9];      // (weight of channel 2e, channel 2e+1) per tap
#pragma unroll
  for (int e = 0; e < 8; ++e) bias[e] = __ldg(b + pl * 8 + e);
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int t = 0; t < 9; ++t) w2[e][t] = f2_pack(__ldg(w + (pl * 8 + 2 * e) * 9 + t), __ldg(w + (pl * 8 + 2 * e + 1) * 9 + t));
  const float* xi = x + (long long)n * H * W;
  __nv_bfloat16* plane = out + ((long long)n * (cout >> 3) + pl) * g.PL * 8;
  const int wq = W >> 2, nq = H * wq;
  float s4[4] = {0.f, 0.f, 0.f, 0.f};
  auto load_patch = [&](int q, float (&xv)[3][6]) {
    const int h = q / wq, w0 = (q - h * wq) << 2;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hh = h + r - 1;
      const bool rowok = q < nq && hh >= 0 && hh < H;
      const float* xr = xi + (long long)hh * W + w0;
      float4 mid = make_float4(0.f, 0.f, 0.f, 0.f);
      if (rowok) mid = __ldg(reinterpret_cast<const float4*>(xr));
      xv[r][0] = (rowok && w0 > 0) ? __ldg(xr - 1) : 0.f;
      xv[r][1] = mid.x; xv[r][2] = mid.y; xv[r][3] = mid.z; xv[r][4] = mid.w;
      xv[r][5] = (rowok && w0 + 4 < W) ? __ldg(xr + 4) : 0.f;
    }
  };
  float xn[3][6];  // next group's patch, fetched while the current one is being multiplied
  load_patch(blockIdx.x * CIQ_ITER * 256 + threadIdx.x, xn);
#pragma unroll 1
  for (int it = 0; it < CIQ_ITER; ++it) {
    const int q = (blockIdx.x * CIQ_ITER + it) * 256 + threadIdx.x;
    if (q >= nq) break;
    const int h = q / wq, w0 = (q - h * wq) << 2;
    float xv[3][6];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) xv[r][c] = xn[r][c];
    if (it + 1 < CIQ_ITER) load_patch(q + 256, xn);
    // channel pairs on packed fp32 lanes (FFMA2): 144 + 36 issue slots per 4 pixels instead of 288; each lane is an
    // IEEE fma in the same order as conv_in_kernel, so the outputs stay bit-identical
    f32x2_t acc2[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc2[u][e] = f2_pack(bias[2 * e], bias[2 * e + 1]);
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float xs = xv[t / 3][u + t % 3];
        const f32x2_t x2 = f2_pack(xs, xs);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc2[u][e] = f2_fma(x2, w2[e][t], acc2[u][e]);
      }
    float acc[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = f2_unpack(acc2[u][e]);
        acc[u][2 * e] = f.x; acc[u][2 * e + 1] = f.y;
      }
    __nv_bfloat16* dst = plane + (long long)(g.lead + h * g.Wp + w0) * 8;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float* a = acc[u];
      uint4 o;
      o.x = pack_bf16x2(a[0], a[1]); o.y = pack_bf16x2(a[2], a[3]);
      o.z = pack_bf16x2(a[4], a[5]); o.w = pack_bf16x2(a[6], a[7]);
      *reinterpret_cast<uint4*>(dst + u * 8) = o;
      s4[0] += a[0] + a[1] + a[2] + a[3];
      s4[1] += a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3];
      s4[2] += a[4] + a[5] + a[6] + a[7];
      s4[3] += a[4] * a[4] + a[5] * a[5] + a[6] * a[6] + a[7] * a[7];
    }
  }
  if (stats) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int sh = 16; sh >= 1; sh >>= 1) s4[k] += __shfl_xor_sync(0xffffffffu, s4[k], sh);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[warp][0] = s4[0]; red[warp][1] = s4[1]; red[warp][2] = s4[2]; red[warp][3] = s4[3]; }
    __syncthreads();
    if (threadIdx.x < 4) {
      float t = 0.f;
      for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
      stat_t* dst = stats + ((long long)n * (cout >> 2) + pl * 2 + (threadIdx.x >> 1)) * 2 + (threadIdx.x & 1);
      atomicAdd(dst, (stat_t)t);
    }
  }
}

cudaError_t launch_conv_in(const float* x, const float* w, const float* b, int N, int cin, int H, int W, int cout,
                           __nv_bfloat16* out, stat_t* stats, cudaStream_t s) {
  if (cin == 1 && (W & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const int nq = H * (W >> 2);
    dim3 grid((nq + 256 * CIQ_ITER - 1) / (256 * CIQ_ITER), cout >> 3, N);
    conv_in_c1_kernel<<<grid, 256, 0, s>>>(x, w, b, N, H, W, cout, out, stats);
    return cudaGetLastError();
  }
  dim3 grid((H * W + 256 * CI_PIX - 1) / (256 * CI_PIX), cout >> 3, N);
  conv_in_kernel<<<grid, 256, 0, s>>>(x, w, b, N, cin, H, W, cout, out, stats);
  return cudaGetLastError();
}

// ------------------------------------------------------------- conv_norm_out + SiLU + conv_out + scheduler step
// HBM-read bound: the kernel streams the raw 128-channel tensor once (halo 1.27x) and writes one fp32 plane.
// Persistent CTAs (2 per SM) walk 16 x 16 output tiles; per tile the 18 x 18 x C halo goes global -> shared memory with
// 16-byte cp.async copies (all of a tile's bytes in flight at once, zero-filled outside the image), is normalised +
// SiLU'd in place (bf16), and the 3x3 conv runs on the warp-level tensor cores (mma.sync m16n8k16: M = 16 pixels of a tile
// row, N = cout padded to 8, K = 16 channels per tap and k-step).  Weight fragments are built once per CTA.
constexpr int CO_TILE = 16;
constexpr int CO_HALO = CO_TILE + 2;
constexpr int CO_MAXOUT = 4;
constexpr int CO_CTAS_PER_SM = 2;

__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;   // src-size 0: nothing is read, the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__global__ void __launch_bounds__(256, CO_CTAS_PER_SM) conv_out_kernel(const ConvOutParams p) {
  extern __shared__ __align__(16) uint8_t osm[];
  const int planes = p.C >> 3;
  constexpr int HV = CO_HALO * CO_HALO;                                         // vectors per plane of the halo tile
  uint4* act = reinterpret_cast<uint4*>(osm);                                   // [planes][324] 16 B vectors
  uint2* wfrag = reinterpret_cast<uint2*>(osm + (size_t)planes * HV * 16);      // [9][C/16][32] B fragments
  float2* ssm = reinterpret_cast<float2*>(wfrag + 9 * (p.C >> 4) * 32);         // [C] (scale, shift) of the current sample
  float* wsm = reinterpret_cast<float*>(act);                                   // [cout][C][9] fp32 weights: build only, aliases the tile
  const Geom g = make_geom(p.N, p.H, p.W);
  const int ksteps = p.C >> 4;
  const int tiles_x = (p.W + CO_TILE - 1) / CO_TILE, tiles_y = (p.H + CO_TILE - 1) / CO_TILE;
  const int tiles_img = tiles_x * tiles_y, ntiles = tiles_img * p.N;

  // weights: fp32 [cout][C][3][3] -> per (tap, 16-channel k-step) the m16n8k16 B fragment (k = channel, n = cout padded
  // to 8): lane (g, tq) holds (ch 2tq, 2tq+1 | ch 8+2tq, 9+2tq) of output channel g, zero for g >= cout
  for (int i = threadIdx.x; i < p.cout * p.C * 9; i += blockDim.x) wsm[i] = __ldg(p.w + i);
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * ksteps * 32; i += blockDim.x) {
    const int ln = i & 31, ks = (i >> 5) % ksteps, t = i / (32 * ksteps);
    const int co = ln >> 2, tq = ln & 3;
    uint2 bf = make_uint2(0u, 0u);
    if (co < p.cout) {
      const float* wp = wsm + ((long long)co * p.C + ks * 16 + 2 * tq) * 9 + t;
      bf.x = pack_bf16x2(wp[0], wp[9]);
      bf.y = pack_bf16x2(wp[72], wp[81]);
    }
    wfrag[i] = bf;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
  const uint32_t act_s = smem_u32(act);
  const uint32_t* act32 = reinterpret_cast<const uint32_t*>(act);
  const int total = planes * HV;
  int cur_n = -1;

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int n = tile / tiles_img, tr = tile - n * tiles_img;
    const int ty = tr / tiles_x, tx = tr - ty * tiles_x;
    const int h0 = ty * CO_TILE, w0 = tx * CO_TILE;
    __syncthreads();                       // the previous tile's MMAs have read `act` (and wfrag / ssm are complete)
    // ---- halo tile: every vector of the tile in flight at once
    const __nv_bfloat16* img = p.src + (long long)n * planes * g.PL * 8;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int pl = i / HV, hp = i - pl * HV;
      const int hy = hp / CO_HALO, hx = hp - hy * CO_HALO;
      const int h = h0 + hy - 1, w = w0 + hx - 1;
      const bool inb = h >= 0 && h < p.H && w >= 0 && w < p.W;
      const __nv_bfloat16* sp = img + ((long long)pl * g.PL + g.lead + (inb ? h * g.Wp + w : 0)) * 8;
      cp_async16_zfill(act_s + (uint32_t)i * 16u, sp, inb);
    }
    if (n != cur_n) {                      // per-sample GroupNorm scale / shift
      cur_n = n;
      if (p.ss) {
        for (int c = threadIdx.x; c < p.C; c += blockDim.x) ssm[c] = __ldg(p.ss + (long long)n * p.C + c);
      } else {                             // stand-alone use: finalize the statistics here
        const int cpg = p.C / p.groups;
        for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
          const int gi = c / cpg;
          double sm = 0., sq = 0.;
          for (int cc = gi * cpg; cc < (gi + 1) * cpg; cc += 4) {
            const stat_t* st = p.stats + ((long long)n * (p.C >> 2) + (cc >> 2)) * 2;
            sm += st[0];
            sq += st[1];
          }
          const double cnt = (double)cpg * (double)p.H * (double)p.W;
          const double mean = sm / cnt;
          const float rstd = (float)(1.0 / sqrt(fmax(sq / cnt - mean * mean, 0.) + (double)p.eps));
          const float sc = p.gamma[c] * rstd;
          ssm[c] = make_float2(sc, p.beta[c] - (float)mean * sc);
        }
      }
    }
    cp_async_wait_all();
    __syncthreads();
    // ---- GroupNorm + SiLU in place (zero outside the image: the conv pads the *activated* tensor)
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int pl = i / HV, hp = i - pl * HV;
      const int hy = hp / CO_HALO, hx = hp - hy * CO_HALO;
      const int h = h0 + hy - 1, w = w0 + hx - 1;
      if (h < 0 || h >= p.H || w < 0 || w >= p.W) continue;
      const uint4 v = act[i];
      const uint32_t uu[4] = {v.x, v.y, v.z, v.w};
      uint32_t r[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_bf16x2(uu[e]);
        const float2 s0 = ssm[pl * 8 + 2 * e], s1 = ssm[pl * 8 + 2 * e + 1];
        r[e] = pack_bf16x2(silu_tanh(fmaf(f.x, s0.x, s0.y)), silu_tanh(fmaf(f.y, s1.x, s1.y)));
      }
      act[i] = make_uint4(r[0], r[1], r[2], r[3]);
    }
    __syncthreads();
    // ---- implicit GEMM: warp w owns tile rows 2w and 2w+1; A fragments are 32-bit reads of the activated halo tile
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    for (int ks = 0; ks < ksteps; ++ks) {
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        const int kh = t / 3, kw = t - kh * 3;
        const uint2 bf = wfrag[(t * ksteps + ks) * 32 + lane];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int v0 = (2 * ks) * HV + (2 * warp + r + kh) * CO_HALO + gq + kw;  // 16-byte vector index
          const uint32_t a0 = act32[v0 * 4 + tq], a1 = act32[(v0 + 8) * 4 + tq];
          const uint32_t a2 = act32[(v0 + HV) * 4 + tq], a3 = act32[(v0 + HV + 8) * 4 + tq];
          asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                       : "+f"(acc[r][0]), "+f"(acc[r][1]), "+f"(acc[r][2]), "+f"(acc[r][3])
                       : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(bf.x), "r"(bf.y));
        }
      }
    }
    // accumulator (r, 2j + cc) = pixel (row 2w + r, column gq + 8j), output channel 2tq + cc
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int h = h0 + 2 * warp + r, w = w0 + gq + 8 * j;
        if (h >= p.H || w >= p.W) continue;
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int co = 2 * tq + cc;
          if (co >= p.cout) continue;
          const float e = acc[r][2 * j + cc] + p.b[co];
          const long long idx = (((long long)n * p.cout + co) * p.H + h) * p.W + w;
          if (p.eps_out) p.eps_out[idx] = e;
          if (p.x_out) {
            const StepCoef cf = p.coef_dev ? *p.coef_dev : p.coef;
            const float xv = p.x[idx];
            float x0 = (xv - cf.sqrt_1m_at * e) * cf.inv_sqrt_at;
            if (cf.do_clip) x0 = fminf(fmaxf(x0, -cf.clip), cf.clip);
            float rr = cf.c_x0 * x0 + cf.c_xt * xv + cf.c_eps * e;
            if (p.z) rr += cf.c_z * p.z[idx];
            p.x_out[idx] = rr;
          }
        }
      }
  }
}

cudaError_t launch_conv_out(const ConvOutParams& p, cudaStream_t s) {
  if (p.cout > CO_MAXOUT || (p.C & 15)) return cudaErrorInvalidValue;
  const size_t smem = (size_t)(p.C >> 3) * CO_HALO * CO_HALO * 16 + (size_t)9 * (p.C >> 4) * 32 * sizeof(uint2) +
                      (size_t)p.C * sizeof(float2);
  static size_t smem_set = 0;
  static int sms = 0;
  if (smem > smem_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    smem_set = smem;
  }
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const int ntiles = ((p.W + CO_TILE - 1) / CO_TILE) * ((p.H + CO_TILE - 1) / CO_TILE) * p.N;
  const int grid = ntiles < sms * CO_CTAS_PER_SM ? ntiles : sms * CO_CTAS_PER_SM;
  conv_out_kernel<<<grid, 256, smem, s>>>(p);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ resampling
// dst4: four PF8 tensors (N, C, H/2, W/2) back to back, index a*2+b holds x[2h'+a, 2w'+b]
__global__ void parity_split_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst4, int N,
                                    int C, int H, int W) {
  const int Ho = H >> 1, Wo = W >> 1;
  const Geom gi = make_geom(N, H, W), go = make_geom(N, Ho, Wo);
  const int pidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (pidx >= Ho * Wo) return;
  const int ho = pidx / Wo, wo = pidx - ho * Wo;
  const long long plane = (long long)blockIdx.z * (C >> 3) + blockIdx.y;
  const long long tsz = (long long)N * (C >> 3) * go.PL * 8;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const uint4 v = *reinterpret_cast<const uint4*>(
          src + (plane * gi.PL + gi.lead + (2 * ho + a) * gi.Wp + 2 * wo + b) * 8);
      *reinterpret_cast<uint4*>(dst4 + (a * 2 + b) * tsz + (plane * go.PL + go.lead + ho * go.Wp + wo) * 8) = v;
    }
}
cudaError_t launch_parity_split(const __nv_bfloat16* src, __nv_bfloat16* dst4, int N, int C, int H, int W, cudaStream_t s) {
  dim3 grid(((H / 2) * (W / 2) + 255) / 256, C >> 3, N);
  parity_split_kernel<<<grid, 256, 0, s>>>(src, dst4, N, C, H, W);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ layout conversion
__global__ void nchw_to_pf8_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, int N, int C, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int pidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (pidx >= H * W) return;
  const int h = pidx / W, w = pidx - h * W;
  const int pl = blockIdx.y, n = blockIdx.z;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = src[(((long long)n * C + pl * 8 + e) * H + h) * W + w];
  uint4 o;
  o.x = pack_bf16x2(v[0], v[1]); o.y = pack_bf16x2(v[2], v[3]);
  o.z = pack_bf16x2(v[4], v[5]); o.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(dst + (((long long)n * (C >> 3) + pl) * g.PL + g.lead + h * g.Wp + w) * 8) = o;
}
cudaError_t launch_nchw_to_pf8(const float* src, __nv_bfloat16* dst, int N, int C, int H, int W, cudaStream_t s) {
  dim3 grid((H * W + 255) / 256, C >> 3, N);
  nchw_to_pf8_kernel<<<grid, 256, 0, s>>>(src, dst, N, C, H, W);
  return cudaGetLastError();
}
__global__ void pf8_to_nchw_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, int N, int C, int H, int W) {
  const Geom g = make_geom(N, H, W);
  const int pidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (pidx >= H * W) return;
  const int h = pidx / W, w = pidx - h * W;
  const int pl = blockIdx.y, n = blockIdx.z;
  const uint4 v = *reinterpret_cast<const uint4*>(src + (((long long)n * (C >> 3) + pl) * g.PL + g.lead + h * g.Wp + w) * 8);
  const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack_bf16x2(u[e]);
    dst[(((long long)n * C + pl * 8 + 2 * e) * H + h) * W + w] = f.x;
    dst[(((long long)n * C + pl * 8 + 2 * e + 1) * H + h) * W + w] = f.y;
  }
}
cudaError_t launch_pf8_to_nchw(const __nv_bfloat16* src, float* dst, int N, int C, int H, int W, cudaStream_t s) {
  dim3 grid((H * W + 255) / 256, C >> 3, N);
  pf8_to_nchw_kernel<<<grid, 256, 0, s>>>(src, dst, N, C, H, W);
  return cudaGetLastError();
}


// ------------------------------------------------------------------------------------ standalone quad stats
// (the hot path gets these from the producing conv's epilogue; this kernel serves tensors that arrive from
// outside, e.g. the op-level GroupNorm entry point)
__global__ void __launch_bounds__(256) quad_stats_kernel(const __nv_bfloat16* __restrict__ src, stat_t* __restrict__ stats,
                                                         int N, int C, int H, int W) {
  __shared__ float red[8][4];
  const Geom g = make_geom(N, H, W);
  const int pl = blockIdx.y, n = blockIdx.z;
  const __nv_bfloat16* sp = src + ((long long)n * (C >> 3) + pl) * g.PL * 8;
  float s4[4] = {0.f, 0.f, 0.f, 0.f};
  for (int pidx = blockIdx.x * blockDim.x + threadIdx.x; pidx < H * W; pidx += gridDim.x * blockDim.x) {
    const int h = pidx / W, w = pidx - h * W;
    const uint4 v = *reinterpret_cast<const uint4*>(sp + (long long)(g.lead + h * g.Wp + w) * 8);
    float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
    s4[0] += a.x + a.y + b.x + b.y;
    s4[1] += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y;
    s4[2] += c.x + c.y + d.x + d.y;
    s4[3] += c.x * c.x + c.y * c.y + d.x * d.x + d.y * d.y;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int sh = 16; sh >= 1; sh >>= 1) s4[k] += __shfl_xor_sync(0xffffffffu, s4[k], sh);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[warp][0] = s4[0]; red[warp][1] = s4[1]; red[warp][2] = s4[2]; red[warp][3] = s4[3]; }
  __syncthreads();
  if (threadIdx.x < 4) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x];
    atomicAdd(stats + ((long long)n * (C >> 2) + pl * 2 + (threadIdx.x >> 1)) * 2 + (threadIdx.x & 1), (stat_t)t);
  }
}
cudaError_t launch_quad_stats(const __nv_bfloat16* src, stat_t* stats, int N, int C, int H, int W, cudaStream_t s) {
  int bx = (H * W + 255) / 256;
  if (bx > 64) bx = 64;
  dim3 grid(bx, C >> 3, N);
  quad_stats_kernel<<<grid, 256, 0, s>>>(src, stats, N, C, H, W);
  return cudaGetLastError();
}

__global__ void stats_to_float_kernel(const stat_t* s, float* d, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = (float)s[i];
}
cudaError_t launch_stats_to_float(const stat_t* s, float* d, int n, cudaStream_t st) {
  stats_to_float_kernel<<<(n + 255) / 256, 256, 0, st>>>(s, d, n);
  return cudaGetLastError();
}

// pipeline_audio_diffusion.py:192-194: (x/2+0.5).clamp(0,1) -> *255 -> numpy round (half to even) -> uint8
__global__ void sample_to_u8_kernel(const float* __restrict__ x, uint8_t* __restrict__ img, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = __fadd_rn(__fdiv_rn(x[i], 2.0f), 0.5f);
  v = fminf(fmaxf(v, 0.0f), 1.0f);
  img[i] = (uint8_t)__float2int_rn(__fmul_rn(v, 255.0f));
}
cudaError_t launch_sample_to_u8(const float* x, uint8_t* img, size_t n, cudaStream_t s) {
  sample_to_u8_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, img, n);
  return cudaGetLastError();
}

}  // namespace b200ad
